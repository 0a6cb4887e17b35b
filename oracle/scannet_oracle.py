"""ScanNet frame path restated: utils.box_filter (utils.py:112-208) + dataset.py:208-292, and a seeded writer of
synthetic ScanNet-format sequences.

TEST INFRASTRUCTURE ONLY.  The restatement imports nothing from the reference, so GPU tests can make new cases on
machines without a reference checkout; it is pinned to the reference's own dataset.ScanNet by the goldens of
oracle/make_scannet_golden.py.  The open3d arithmetic comes from oracle/o3d_standin.py (restated, not checked).

Background-class rule for an instance that carries several semantic classes: the reference raises (``ndarray in
list``); here, as in the Replica ingest, the smallest class decides.
"""
from __future__ import annotations

import glob
import os

import cv2
import numpy as np
from scipy import ndimage

from oracle import o3d_standin as o3d

BG_CLASSES = (-1, 0, 1, 3, 16, 41, 232, 21, 161, 128, 21)     # dataset.py:187
MIN_PIXELS = 1500                                            # dataset.py:184
BBOX_SCALE = 0.2                                             # dataset.py:188
VOXEL = 0.01                                                 # utils.py:112


class Track:
    def __init__(self, inst_id, pc, box):
        self.inst_id = inst_id
        self.pc = pc
        self.center, self.R, self.extent = box
        self.cmp_cnt = 0
        self.merge_cnt = 0


def erode13(mask):
    """cv2.erode(mask, ones((5, 5)), iterations=3): a pixel survives iff every in-image pixel within Chebyshev
    distance 6 is set (the constant border does not erode)."""
    return ndimage.minimum_filter(mask.astype(np.uint8), size=13, mode="constant", cval=1).astype(bool)


def enlarge(x0, y0, x1, y1, scale, w, h):
    """utils.enlarge_bbox on python ints (fp64 margins); None when a margin is 0."""
    mx = int(0.5 * scale * (x1 - x0))
    my = int(0.5 * scale * (y1 - y0))
    if mx == 0 or my == 0:
        return None
    return (min(max(x0 - mx, 0), w - 1), min(max(y0 - my, 0), h - 1),
            min(max(x1 + mx, 0), w - 1), min(max(y1 + my, 0), h - 1))


def box_filter(inst, sem, depth, tracks, intr, camera_pose, min_pixels=MIN_PIXELS, voxel=VOXEL, bg=BG_CLASSES):
    """inst: [H, W] int32 ids (already +1); sem: [H, W]; depth: [H, W] f32.  Returns the int64 label image and
    updates ``tracks`` {id: Track}.  Background-class instances are dropped first (dataset.py:252-261)."""
    fx, fy, cx, cy = intr
    labels = np.zeros(depth.shape, np.int64)
    for iid in np.unique(inst):
        m = inst == iid
        if int(sem[m].min()) in bg or iid == 0:
            continue
        pts = o3d.unproject(np.where(m, depth, np.float32(0)), fx, fy, cx, cy, camera_pose)
        if len(pts) <= 10:
            continue
        iid = int(iid)
        tr = tracks.get(iid)
        if tr is not None:
            tr.cmp_cnt += 1
            ins = o3d.inside_box(pts, tr.center, tr.R, tr.extent)
            if not ins.any():
                labels[m] = -1
                continue
            tr.pc = o3d.voxel_down_sample(np.concatenate([tr.pc, pts[ins]]), voxel)
            try:
                tr.center, tr.R, tr.extent = o3d.obb_from_points(tr.pc)
            except RuntimeError:
                labels[m] = -1
                continue
            valid = m & (depth > 0)
            diff = np.zeros_like(m)
            diff[valid] = ~ins
            labels[m] = iid
            labels[diff] = -1
        else:
            small = erode13(m)
            if small.sum() < min_pixels:
                continue
            pe = o3d.unproject(np.where(small, depth, np.float32(0)), fx, fy, cx, cy, camera_pose)
            pc = o3d.voxel_down_sample(pe, voxel)
            try:
                box = o3d.obb_from_points(pc)
            except RuntimeError:
                continue
            tracks[iid] = Track(iid, pc, box)
            labels[m] = iid
    return labels


def finalize(labels, bbox_scale=BBOX_SCALE):
    """dataset.py:263-281: per-label pixel box, enlarged; None -> relabel 0; 0 is the full frame."""
    H, W = labels.shape
    bbox = {}
    for lab in np.unique(labels):
        m = labels == lab
        v, u = np.nonzero(m)
        if len(u) == 0:
            continue
        e = enlarge(int(u.min()), int(v.min()), int(u.max()) + 1, int(v.max()) + 1, bbox_scale, W, H)
        if e is None:
            labels[m] = 0
        else:
            bbox[int(lab)] = np.array([e[0], e[2], e[1], e[3]], np.int64)
    bbox[0] = np.array([0, W, 0, H], np.int64)
    return labels, bbox


# ---- ScanNet-format files --------------------------------------------------------------------------------------

def _sorted(root, sub, ext):
    return sorted(glob.glob(os.path.join(root, sub, "*" + ext)), key=lambda x: int(os.path.basename(x)[:-4]))


def load_poses(root):
    return [np.loadtxt(p).reshape(4, 4) for p in _sorted(root, "pose", ".txt")]


def load_frame(root, index, W, H, edge, depth_scale, max_depth, poses, imap_mode=False):
    """dataset.py:208-262's host part: decode, resize, edge crop, depth scale / filter; the inf-pose skip.
    Returns (rgb [H', W', 3] u8, depth [H', W'] f32, T, inst [H', W'] int32 (+1), sem) or None."""
    n = len(poses)
    while np.any(np.isinf(poses[index])):
        if index + 1 == n:
            return None
        index += 1
    color = cv2.cvtColor(cv2.imread(_sorted(root, "color", ".jpg")[index]).astype(np.uint8), cv2.COLOR_BGR2RGB)
    depth = cv2.imread(_sorted(root, "depth", ".png")[index], cv2.IMREAD_UNCHANGED).astype(np.float32)
    depth = np.nan_to_num(depth, nan=0.)
    h, w = depth.shape
    color = cv2.resize(color, (w, h), interpolation=cv2.INTER_LINEAR)
    sl = (slice(edge, -edge), slice(edge, -edge)) if edge else (slice(None), slice(None))
    color, depth = color[sl], depth[sl]
    depth = depth.astype(np.float32) * depth_scale
    depth[depth > max_depth] = 0.
    if imap_mode:
        return color, depth, poses[index], None, None
    inst = cv2.resize(cv2.imread(_sorted(root, "instance-filt", ".png")[index], cv2.IMREAD_UNCHANGED), (w, h),
                      interpolation=cv2.INTER_NEAREST).astype(np.int32)
    sem = cv2.resize(cv2.imread(_sorted(root, "label-filt", ".png")[index], cv2.IMREAD_UNCHANGED), (w, h),
                     interpolation=cv2.INTER_NEAREST)
    return color, depth, poses[index], inst[sl] + 1, sem[sl]


class Sequence:
    """The restated dataset.ScanNet: one tracking state, frames fed in any order the caller chooses."""

    def __init__(self, root, W=620, H=460, edge=10, depth_scale=1 / 1000.0, max_depth=6.0, imap_mode=False):
        self.root, self.W, self.H, self.edge = root, W, H, edge
        self.depth_scale, self.max_depth, self.imap_mode = depth_scale, max_depth, imap_mode
        k = np.loadtxt(os.path.join(root, "intrinsic", "intrinsic_depth.txt"))
        self.intr = (k[0, 0], k[1, 1], k[0, 2] - edge, k[1, 2] - edge)
        self.poses = load_poses(root)
        self.tracks = {}

    def __len__(self):
        return len(self.poses)

    def __getitem__(self, index):
        fr = load_frame(self.root, index, self.W, self.H, self.edge, self.depth_scale, self.max_depth, self.poses,
                        self.imap_mode)
        if fr is None:
            return None
        color, depth, T, inst, sem = fr
        if self.imap_mode:
            labels = np.zeros(depth.shape, np.int32)
            bbox = {0: np.array([0, labels.shape[1], 0, labels.shape[0]], np.int64)}
        else:
            camera_pose = np.linalg.inv(np.linalg.inv(T))          # open3d inverts the T_CW it is handed
            labels = box_filter(inst, sem, depth, self.tracks, self.intr, camera_pose)
            labels, bbox = finalize(labels)
        return {"image": color.transpose(1, 0, 2), "depth": depth.transpose(1, 0), "T": T, "T_obj": np.eye(4),
                "obj": labels.transpose(1, 0), "bbox_dict": bbox}


# ---- seeded synthetic ScanNet-format sequence ------------------------------------------------------------------

INTR = np.array([[577.87, 0, 319.5, 0], [0, 577.87, 239.5, 0], [0, 0, 1, 0], [0, 0, 0, 1]])


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def _pose(i, n):
    """Camera-to-world pose of frame i: a slow sideways move and yaw (camera z forward, y down)."""
    yaw = 0.08 * np.sin(2 * np.pi * i / max(n, 1))
    c, s = np.cos(yaw), np.sin(yaw)
    T = np.eye(4)
    T[:3, :3] = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
    T[:3, 3] = [0.05 * i - 0.2, 0.01 * i, 0.02 * i]
    return T


def _render(T, objs, rng, Wd=640, Hd=480):
    """Ray-cast floor (y = 1.2, class 3), back wall (z = 4.5, class 1) and ellipsoids.  Returns depth [H, W] f64
    (0 = no hit), instance and class images."""
    K = INTR
    v, u = np.mgrid[0:Hd, 0:Wd].astype(np.float64)
    dc = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1)     # camera z = 1
    R, t = T[:3, :3], T[:3, 3]
    dw = dc @ R.T
    best = np.full((Hd, Wd), np.inf)
    inst = np.zeros((Hd, Wd), np.int32)
    cls = np.zeros((Hd, Wd), np.int32)
    for (axis, val, iid, c) in ((1, 1.2, 1, 3), (2, 4.5, 2, 1)):
        with np.errstate(divide="ignore", invalid="ignore"):
            s = (val - t[axis]) / dw[..., axis]
        hit = (s > 0.1) & (s < best)
        best[hit], inst[hit], cls[hit] = s[hit], iid, c
    for o in objs:
        Ro, r = o["R"], np.asarray(o["radii"])
        oc = (t - o["center"]) @ Ro / r                                  # ellipsoid frame, unit sphere
        od = (dw @ Ro) / r
        a = (od * od).sum(-1)
        b = 2 * (od * oc).sum(-1)
        c = (oc * oc).sum() - 1
        disc = b * b - 4 * a * c
        with np.errstate(invalid="ignore"):
            s = (-b - np.sqrt(disc)) / (2 * a)
        hit = (disc > 0) & (s > 0.1) & (s < best)
        best[hit], inst[hit], cls[hit] = s[hit], o["id"], o["cls"]
    depth = np.where(np.isfinite(best), best, 0.0)                       # camera z (dc has z = 1)
    depth = np.where(depth > 0, depth + rng.normal(0, 0.002, depth.shape), 0.0)
    return depth, inst, cls


def default_objects(rng, n_extra=0, id_base=10):
    """Objects of the branch-covering sequence.  ids are instance-filt values (the loader adds 1)."""
    objs = [
        dict(name="A", id=id_base + 0, cls=5, center=[0.0, 0.3, 2.2], radii=[0.45, 0.3, 0.35]),   # new, then merged
        dict(name="B", id=id_base + 1, cls=7, center=[-1.55, 0.2, 2.6], radii=[0.4, 0.35, 0.3]),  # cut by the border
        dict(name="C", id=id_base + 2, cls=9, center=[0.9, 0.9, 2.5], radii=[0.07, 0.06, 0.05]),  # small -> 0
        dict(name="D", id=id_base + 3, cls=11, center=[0.3, -0.9, 6.8], radii=[0.5, 0.4, 0.3]),   # depth > max -> 0
        dict(name="E", id=id_base + 4, cls=12, center=[0.75, -0.45, 2.4], radii=[0.25, 0.3, 0.2]), # hull fails -> 0
        dict(name="G", id=id_base + 5, cls=14, center=[-0.6, -0.5, 3.0], radii=[0.25, 0.2, 0.3]), # moves away later
        dict(name="H", id=id_base + 6, cls=14, center=[0.8, 0.6, 3.6], radii=[0.3, 0.25, 0.25]),  # G's second home
    ]
    for k in range(n_extra):
        objs.append(dict(name=f"X{k}", id=id_base + 7 + k, cls=5 + (k % 3) * 2,
                         center=[rng.uniform(-1.6, 1.6), rng.uniform(-0.8, 0.9), rng.uniform(1.8, 4.0)],
                         radii=list(rng.uniform(0.08, 0.35, 3))))
    for o in objs:
        o["R"] = _rot(rng)
        o["center"] = np.asarray(o["center"], np.float64)
    return objs


def write_sequence(root, seed=0, n_frames=10, n_extra=0, id_base=10, inf_frame=4, color_size=(1296, 968)):
    """Write color/*.jpg (color_size, resized by the loader), depth/*.png (u16 mm), instance-filt/*.png and
    label-filt/*.png (u16), pose/*.txt and intrinsic/intrinsic_depth.txt.  Frame script (default objects):
      every frame : A (new, then tracked / merged, with diff pixels), B (cut by the left border), C (small),
                    D (beyond max_depth), E (depth only on a 4-px rim: > 10 points, < 4 eroded points)
      frames < 5  : G at its own place (new, then tracked);  frames >= 5: G's id painted on H (far from its box: -1)
      frame 7     : only G's id, as a 6-px strip on the wall (whole mask -1, then too thin: 0), plus C
      frame 8     : A's id only on an 8-px column of A (merged, then too narrow: 0)
      inf_frame   : pose with inf (the loader skips to the next frame)"""
    rng = np.random.default_rng(seed)
    objs = default_objects(rng, n_extra, id_base)
    by = {o["name"]: o for o in objs}
    for sub in ("color", "depth", "instance-filt", "label-filt", "pose", "intrinsic"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    np.savetxt(os.path.join(root, "intrinsic", "intrinsic_depth.txt"), INTR)
    scripted = n_extra == 0
    for i in range(n_frames):
        T = _pose(i, n_frames)
        vis = [o for o in objs if o["name"] not in ("G", "H")]
        if scripted and i == 7:
            vis = [by["C"]]
        if i < 5:
            vis.append(by["G"])
        elif scripted and i != 7:
            vis.append(dict(by["H"], id=by["G"]["id"]))
        depth, inst, cls = _render(T, vis, rng)
        if scripted and i == 7:
            inst[150:260, 300:306], cls[150:260, 300:306] = by["G"]["id"], by["G"]["cls"]
        if scripted and i == 8:
            a = inst == by["A"]["id"]
            cols = np.nonzero(a.any(0))[0]
            c0 = cols[len(cols) // 2]
            keep = a.copy()
            keep[:, :c0] = False
            keep[:, c0 + 8:] = False
            inst[a & ~keep], cls[a & ~keep] = 0, 0
        e = inst == by["E"]["id"]
        if e.any():                                      # E: depth only on a rim of 4 px, plus 3 deep pixels
            deep = ndimage.minimum_filter(e.astype(np.uint8), size=9, mode="constant", cval=0).astype(bool)
            keep = np.argwhere(ndimage.minimum_filter(e.astype(np.uint8), size=31, mode="constant", cval=0))
            depth[deep] = 0.0
            for (r, c) in keep[:: max(len(keep) // 3, 1)][:3]:
                depth[r, c] = 2.4
        dmm = np.clip(np.round(depth * 1000.0), 0, 65535).astype(np.uint16)
        cv2.imwrite(os.path.join(root, "depth", f"{i}.png"), dmm)
        cv2.imwrite(os.path.join(root, "instance-filt", f"{i}.png"), inst.astype(np.uint16))
        cv2.imwrite(os.path.join(root, "label-filt", f"{i}.png"), cls.astype(np.uint16))
        hue = (inst * 37 % 180).astype(np.uint8)
        hsv = np.stack([hue, np.full_like(hue, 200), (80 + 150 * np.exp(-depth / 3)).astype(np.uint8)], -1)
        bgr = cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR)
        cv2.imwrite(os.path.join(root, "color", f"{i}.jpg"), cv2.resize(bgr, color_size, interpolation=cv2.INTER_LINEAR))
        if i == inf_frame:
            T = T.copy()
            T[0, 0] = np.inf
        with open(os.path.join(root, "pose", f"{i}.txt"), "w") as f:
            f.write("\n".join(" ".join(repr(float(x)) for x in row) for row in T) + "\n")
    return objs


def run(root, order=None, n_trackers=1, **kw):
    """Feed frames to ``n_trackers`` restated datasets round-robin (frame i -> tracker i % n); per frame returns
    the sample and a snapshot of that tracker's tracks."""
    seqs = [Sequence(root, **kw) for _ in range(n_trackers)]
    out = []
    for i in (order if order is not None else range(len(seqs[0]))):
        s = seqs[i % n_trackers]
        smp = s[i]
        snap = {k: (t.center.copy(), t.R.copy(), t.extent.copy(), len(t.pc), t.cmp_cnt) for k, t in s.tracks.items()}
        out.append((smp, snap))
    return out
