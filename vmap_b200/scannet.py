"""ScanNet sequences: GPU instance association (utils.box_filter, utils.py:112-208) and a ScanNet loader
(dataset.py:150-292) whose per-frame tracking runs on the GPU (vmb_assoc_*, csrc/k_assoc.cuh).

``InstanceTracker`` holds one sequence's tracking state: per-instance fp64 point clouds on the device, the box table,
``cmp_cnt`` / ``merge_cnt`` and an ``inst_dict`` view shaped like the reference's (``InstData`` with ``inst_id``,
``bbox3D`` as ``utils.BoundingBox``, ``pc`` as a device [n, 3] fp64 tensor).  Per frame it makes two host syncs: one
after voxel downsampling (the oriented box of every changed cloud is fitted on the host: qhull via scipy), one for
the 2-D boxes.

``ScanNet(cfg)`` mirrors dataset.ScanNet: same paths, pose loading and inf-pose skip; decode, resize, edge crop and
depth scale / filter stay on the host with the reference's cv2 / numpy calls; association runs on
``cfg.data_device``; there is no ``cv2.imshow``.  ``init_loader(cfg)`` yields its samples in order, decoding ahead on
threads.  By default it reproduces the reference's 4-worker DataLoader, where each worker has its own ``inst_dict``:
frame i is associated by tracker i % 4.  ``multi_worker=False`` uses one tracker, as the single-worker loader does;
``shared_tracker=True`` is the opt-in deviation that tracks all frames with one tracker.

``read_sequence(cfg)`` is the reader for online SLAM (``slam.Slam(assoc=...)``): every frame in order with its GT pose,
which may be inf, and no association (the SLAM loop runs it at the tracked pose).
"""
from __future__ import annotations

import ctypes as C
import glob
import os
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch
from scipy.spatial import ConvexHull, QhullError

from . import _lib
from .mesh import _Kernels
from .utils import BoundingBox

BG_CLASSES = (-1, 0, 1, 3, 16, 41, 232, 21, 161, 128, 21)     # dataset.py:187
MIN_PIXELS = 1500                                            # dataset.py:184
BBOX_SCALE = 0.2                                             # dataset.py:188
N_WORKERS = 4                                                # dataset.py:52
MERGE, NEW, NEG = 1, 2, 3                                    # VMB_ASSOC_MERGE / NEW / NEG
FINAL_ZERO, FINAL_ID, FINAL_NEG = 0, 1, 2                    # VMB_ASSOC_FINAL_*


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _dot3(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def obb_from_points(points):
    """open3d 0.16 OrientedBoundingBox.create_from_points: convex hull vertices, raw-moment mean / covariance,
    eigenvectors by descending eigenvalue (open3d's three swaps), R[:, 2] = R[:, 0] x R[:, 1], AABB in that frame.
    Returns (center, R, extent); raises RuntimeError where qhull fails (open3d's RuntimeError)."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    try:
        hull = ConvexHull(p)
    except (QhullError, ValueError) as e:
        raise RuntimeError(f"qhull: {e}") from None
    hv = p[hull.vertices]
    n = float(len(hv))
    m = hv.sum(axis=0) / n
    xx = np.stack([hv[:, 0] * hv[:, 0], hv[:, 0] * hv[:, 1], hv[:, 0] * hv[:, 2],
                   hv[:, 1] * hv[:, 1], hv[:, 1] * hv[:, 2], hv[:, 2] * hv[:, 2]], axis=1).sum(axis=0) / n
    cov = np.array([[xx[0] - m[0] * m[0], xx[1] - m[0] * m[1], xx[2] - m[0] * m[2]],
                    [0.0, xx[3] - m[1] * m[1], xx[4] - m[1] * m[2]],
                    [0.0, 0.0, xx[5] - m[2] * m[2]]])
    cov[1, 0], cov[2, 0], cov[2, 1] = cov[0, 1], cov[0, 2], cov[1, 2]
    evals, R = np.linalg.eigh(cov)
    evals, R = evals.copy(), R.copy()
    for a, b in ((1, 0), (2, 0), (2, 1)):
        if evals[a] > evals[b]:
            evals[[a, b]] = evals[[b, a]]
            R[:, [a, b]] = R[:, [b, a]]
    R[:, 0] /= np.sqrt(_dot3(R[:, 0], R[:, 0]))
    R[:, 1] /= np.sqrt(_dot3(R[:, 1], R[:, 1]))
    R[:, 2] = np.cross(R[:, 0], R[:, 1])
    d = hv - m
    local = np.stack([_dot3(d, R[:, j]) for j in range(3)], axis=1)
    lo, hi = local.min(axis=0), local.max(axis=0)
    c_loc = (lo + hi) * 0.5
    center = np.array([_dot3(R[r], c_loc) for r in range(3)]) + m
    return center, R, hi - lo


def box_row(center, R, extent):
    """One row of the device box table: tracked flag, center, the half axes R[:, j] * extent[j] / 2, their squared
    lengths (open3d's inclusive test |d . dx| <= dx . dx)."""
    row = np.zeros(16, np.float64)
    row[0] = 1.0
    row[1:4] = center
    for j in range(3):
        ax = R[:, j] * (0.5 * extent[j])
        row[4 + 3 * j:7 + 3 * j] = ax
        row[13 + j] = _dot3(ax, ax)
    return row


class InstData:
    """utils.InstData (utils.py:101-109) with the cloud as a device tensor."""

    def __init__(self, inst_id):
        self.bbox3D = None
        self.inst_id = inst_id
        self.class_id = None
        self.pc_sample = None
        self.pc = None
        self.merge_cnt = 0      # box_filter never increments it (utils.py:112-208)
        self.cmp_cnt = 0


class InstanceTracker:
    """Per-sequence association state; ``frame`` runs box_filter + the 2-D box pass of dataset.py for one frame."""

    def __init__(self, fx, fy, cx, cy, device="cuda", min_pixels=MIN_PIXELS, voxel_size=0.01,
                 bbox_scale=BBOX_SCALE, bg_classes=BG_CLASSES, inst_dict=None):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.VmbError("instance association runs on a CUDA device: there is no CPU fallback")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.min_pixels, self.voxel_size, self.bbox_scale = int(min_pixels), float(voxel_size), float(bbox_scale)
        bg = [c for c in bg_classes if c >= 0]
        self.bg = torch.zeros(max(bg) + 1 if bg else 1, dtype=torch.uint8)
        self.bg[bg] = 1
        self.bg = self.bg.to(self.device)
        self.inst_dict = {} if inst_dict is None else inst_dict
        self.last_bbox = None       # the last frame's device box table [max_id + 1, 5] int64 (FrameStore.relabel)
        self._k = _Kernels(self.device)
        self.times = {"classify": 0.0, "voxel": 0.0, "hull": 0.0, "finalize": 0.0}
        self.timing = False

    @property
    def cmp_cnt(self):
        return {k: v.cmp_cnt for k, v in self.inst_dict.items()}

    @property
    def merge_cnt(self):
        return {k: v.merge_cnt for k, v in self.inst_dict.items()}

    def _tick(self, name, t0):
        if self.timing:
            torch.cuda.synchronize(self.device)
            t1 = time.perf_counter()
            self.times[name] += t1 - t0
            return t1
        return t0

    def frame(self, inst, depth, T=None, sem=None, max_id=None, camera_pose=None, relabel=True):
        """inst: [W, H] int32 ids (instance + 1, dataset.py:247; 0 = none), depth: [W, H] f32 metres, sem: optional
        [W, H] int32 classes (an instance whose smallest class is a background class is dropped), T: camera-to-world
        4x4 (open3d is handed inv(T) and inverts it again, so camera_pose = inv(inv(T)) as the reference computes it).
        Returns the device int64 [W, H] label image and ``bbox_dict`` {label: int64 tensor [u_lo, u_hi, v_lo, v_hi]}
        (with relabel=False: box_filter's labels, before the 2-D box pass, and no bbox_dict)."""
        dev = self.device
        inst = torch.as_tensor(inst).to(dev, torch.int32).contiguous()
        depth = torch.as_tensor(depth).to(dev, torch.float32).contiguous()
        W, H = inst.shape
        if max_id is None:
            max_id = int(inst.max()) + 1 if inst.numel() else 1
        max_id = max(int(max_id), 1)
        if camera_pose is None:
            camera_pose = np.linalg.inv(np.linalg.inv(np.asarray(T, np.float64)))
        cls = None
        if sem is not None:
            cls = torch.as_tensor(sem).to(dev, torch.int32).contiguous()
        t0 = time.perf_counter()
        if self.timing:
            torch.cuda.synchronize(dev)
        # device box table and previous clouds of the tracked ids this frame can contain
        boxes = np.zeros((max_id, 16), np.float64)
        cloud_off = np.zeros(max_id, np.int32)
        cloud_cnt = np.zeros(max_id, np.int32)
        pcs, n_pool = [], 0
        for k, d in sorted(self.inst_dict.items()):
            if k < max_id:
                boxes[k] = d._row
                cloud_off[k], cloud_cnt[k] = n_pool, len(d.pc)
                n_pool += len(d.pc)
                pcs.append(d.pc)
        pool = torch.cat(pcs) if pcs else torch.zeros((0, 3), dtype=torch.float64, device=dev)
        boxes_d = torch.from_numpy(boxes).to(dev)
        off_d, cnt_d = torch.from_numpy(cloud_off).to(dev), torch.from_numpy(cloud_cnt).to(dev)
        stats = torch.empty((max_id, 8), dtype=torch.int32, device=dev)
        cloud_out = torch.empty((n_pool + W * H, 3), dtype=torch.float64, device=dev)
        final = torch.zeros(max_id, dtype=torch.int32)
        labels = torch.empty((W, H), dtype=torch.int64, device=dev)
        bbox = torch.empty((max_id + 1, 5), dtype=torch.int64, device=dev)
        a = _lib.AssocArgs()
        a.width, a.height, a.inst, a.cls, a.depth, a.max_id = W, H, _p(inst), _p(cls), _p(depth), max_id
        if cls is not None:
            a.bg_class, a.n_class = _p(self.bg), self.bg.numel()
        a.fx, a.fy, a.cx, a.cy = self.fx, self.fy, self.cx, self.cy
        for i, x in enumerate(np.asarray(camera_pose, np.float64).reshape(16)):
            a.camera_pose[i] = float(x)
        a.min_pixels, a.voxel_size, a.bbox_scale = self.min_pixels, self.voxel_size, self.bbox_scale
        a.boxes, a.pool, a.cloud_off, a.cloud_cnt, a.n_pool = _p(boxes_d), _p(pool), _p(off_d), _p(cnt_d), n_pool
        a.stats, a.cloud_out, a.max_cloud_out = _p(stats), _p(cloud_out), n_pool + W * H
        a.labels, a.bbox, a.relabel = _p(labels), _p(bbox), int(bool(relabel))
        self._k.call("vmb_assoc_classify", a)
        t0 = self._tick("classify", t0)
        self._k.call("vmb_assoc_voxel", a)                      # the frame's first host sync
        st = stats.cpu().numpy()
        nvox = st[:, 7].astype(np.int64)
        offs = np.concatenate([[0], np.cumsum(nvox)])
        host_pts = cloud_out[:int(offs[-1])].cpu().numpy()
        t0 = self._tick("voxel", t0)
        fin = final.numpy()
        for k in np.nonzero(st[:, 6])[0]:
            k, act = int(k), int(st[k, 6])
            if act == NEG:
                self.inst_dict[k].cmp_cnt += 1
                fin[k] = FINAL_NEG
                continue
            lo, hi = int(offs[k]), int(offs[k + 1])
            if act == MERGE:
                d = self.inst_dict[k]
                d.cmp_cnt += 1
                d.pc = cloud_out[lo:hi].clone()                 # the merged cloud stays, even if the fit fails
            try:
                box = obb_from_points(host_pts[lo:hi])
            except RuntimeError:
                fin[k] = FINAL_NEG if act == MERGE else FINAL_ZERO
                continue
            if act == NEW:
                d = InstData(k)
                d.pc = cloud_out[lo:hi].clone()
                self.inst_dict[k] = d
            d.bbox3D = BoundingBox()
            d.bbox3D.center, d.bbox3D.R, d.bbox3D.extent = box
            d._row = box_row(*box)
            fin[k] = FINAL_ID
        t0 = self._tick("hull", t0)
        final_d = final.to(dev)
        a.final_label = _p(final_d)
        self._k.call("vmb_assoc_finalize", a)
        self.last_bbox = bbox
        if not relabel:
            self._tick("finalize", t0)
            return labels, None
        bb = bbox.cpu().numpy()                                 # the frame's second host sync
        bbox_dict = {}
        for i in np.nonzero(bb[:, 0])[0]:
            bbox_dict[int(i) - 1] = torch.from_numpy(bb[i, 1:].copy())
        self._tick("finalize", t0)
        return labels, bbox_dict


# ---- ScanNet loader ---------------------------------------------------------------------------------------------

def _sorted(root, sub, ext):
    return sorted(glob.glob(os.path.join(root, sub, "*" + ext)), key=lambda x: int(os.path.basename(x)[:-4]))


class ScanNet:
    """dataset.ScanNet (dataset.py:150-292) with the association on ``cfg.data_device``."""

    def __init__(self, cfg, n_trackers=1):
        self.imap_mode = cfg.imap_mode
        self.root_dir = cfg.dataset_dir
        self.color_paths = _sorted(self.root_dir, "color", ".jpg")
        self.depth_paths = _sorted(self.root_dir, "depth", ".png")
        self.inst_paths = _sorted(self.root_dir, "instance-filt", ".png")
        self.sem_paths = _sorted(self.root_dir, "label-filt", ".png")
        self.load_poses(os.path.join(self.root_dir, "pose"))
        self.n_img = len(self.color_paths)
        self.depth_scale, self.max_depth = cfg.depth_scale, cfg.max_depth
        self.W, self.H = cfg.W, cfg.H
        self.fx, self.fy, self.cx, self.cy = cfg.fx, cfg.fy, cfg.cx, cfg.cy
        self.edge = cfg.mw
        self.device = torch.device(cfg.data_device)
        self.min_pixels = MIN_PIXELS
        self.background_cls_list = list(BG_CLASSES)
        self.bbox_scale = BBOX_SCALE
        self.trackers = [InstanceTracker(self.fx, self.fy, self.cx, self.cy, self.device, self.min_pixels,
                                         bbox_scale=self.bbox_scale) for _ in range(n_trackers)]
        self.inst_dict = self.trackers[0].inst_dict if self.trackers else {}

    def load_poses(self, path):
        self.poses = []
        for pose_path in _sorted(path, "", ".txt"):
            with open(pose_path) as f:
                ls = [list(map(float, line.split(" "))) for line in f.readlines()]
            self.poses.append(np.array(ls).reshape(4, 4))

    def __len__(self):
        return self.n_img

    def decode(self, index):
        """Host part of dataset.py:208-262 (the reference's own cv2 / numpy calls), with the inf-pose skip."""
        while np.any(np.isinf(self.poses[index])):
            if index + 1 == self.n_img:
                return None
            index += 1
        return self.decode_at(index)

    def decode_at(self, index):
        """``decode`` of frame ``index`` itself, whatever its pose (which may be non-finite)."""
        color = cv2.imread(self.color_paths[index]).astype(np.uint8)
        color = cv2.cvtColor(color, cv2.COLOR_BGR2RGB)
        depth = cv2.imread(self.depth_paths[index], cv2.IMREAD_UNCHANGED).astype(np.float32)
        depth = np.nan_to_num(depth, nan=0.)
        T = self.poses[index]
        H, W = depth.shape
        color = cv2.resize(color, (W, H), interpolation=cv2.INTER_LINEAR)
        e = self.edge
        if e:
            color, depth = color[e:-e, e:-e], depth[e:-e, e:-e]
        depth = depth.astype(np.float32) * self.depth_scale
        depth[depth > self.max_depth] = 0.
        inst = sem = None
        if not self.imap_mode:
            inst = cv2.resize(cv2.imread(self.inst_paths[index], cv2.IMREAD_UNCHANGED), (W, H),
                              interpolation=cv2.INTER_NEAREST).astype(np.int32)
            sem = cv2.resize(cv2.imread(self.sem_paths[index], cv2.IMREAD_UNCHANGED), (W, H),
                             interpolation=cv2.INTER_NEAREST)
            if e:
                inst, sem = inst[e:-e, e:-e], sem[e:-e, e:-e]
            inst = inst + 1
        return color, depth, T, inst, sem

    def associate(self, decoded, tracker=0):
        """Device part: box_filter + the 2-D box pass on tracker ``tracker``; returns the sample dict."""
        if decoded is None:
            return None
        color, depth, T, inst, sem = decoded
        dev = self.device
        depth_t = torch.from_numpy(np.ascontiguousarray(depth.T)).to(dev)
        if self.imap_mode:
            obj = torch.zeros(depth_t.shape, dtype=torch.int32, device=dev)
            bbox_dict = {0: torch.tensor([0, depth.shape[1], 0, depth.shape[0]], dtype=torch.int64)}
        else:
            max_id = int(inst.max()) + 1
            semc = np.clip(sem.astype(np.int64), -1, None).astype(np.int32)
            obj, bbox_dict = self.trackers[tracker].frame(np.ascontiguousarray(inst.T), depth_t, T=T,
                                                          sem=np.ascontiguousarray(semc.T), max_id=max_id)
        return {"image": torch.from_numpy(np.ascontiguousarray(color.transpose(1, 0, 2))),
                "depth": depth_t, "T": torch.from_numpy(np.asarray(T, np.float64)),
                "T_obj": torch.from_numpy(np.identity(4)), "obj": obj, "bbox_dict": bbox_dict}

    def __getitem__(self, index):
        return self.associate(self.decode(index))


class _Loader:
    """In-order iterable over a ScanNet dataset: host decode prefetched on threads, association in this process."""

    def __init__(self, dataset, n_trackers, prefetch=4):
        self.dataset, self.n_trackers, self.prefetch = dataset, n_trackers, prefetch

    def __len__(self):
        return len(self.dataset)

    def __iter__(self):
        ds = self.dataset
        with ThreadPoolExecutor(max_workers=self.prefetch) as pool:
            futs = {}
            for i in range(min(self.prefetch, len(ds))):
                futs[i] = pool.submit(ds.decode, i)
            for i in range(len(ds)):
                nxt = i + self.prefetch
                if nxt < len(ds):
                    futs[nxt] = pool.submit(ds.decode, nxt)
                yield ds.associate(futs.pop(i).result(), i % self.n_trackers)


def init_loader(cfg, multi_worker=True, shared_tracker=False):
    """dataset.init_loader for ScanNet configs.  Frame i is associated by tracker i % 4 with multi_worker=True (the
    reference's four DataLoader workers each keep their own inst_dict), by one tracker with multi_worker=False or
    shared_tracker=True (opt-in: one tracking state for the whole sequence)."""
    if cfg.dataset_format != "ScanNet":
        raise ValueError(f"vmap_b200.scannet.init_loader handles ScanNet configs, not {cfg.dataset_format}")
    n = N_WORKERS if multi_worker and not shared_tracker else 1
    return _Loader(ScanNet(cfg, n_trackers=n), n)


def read_sequence(cfg, frames=None, prefetch=4):
    """The frames of a ScanNet sequence in order, for online SLAM (``slam.Slam(assoc=...)``): no association, and no
    inf-pose skip (GT is only used to score a trajectory, so a frame whose GT pose is invalid is still a frame).  Host
    decode as ``ScanNet.decode`` (resize, edge crop, depth scale / filter), ``prefetch`` frames ahead on threads.
    Yields per frame a dict: ``index``, ``rgb`` [W, H, 3] uint8, ``depth`` [W, H] f32 metres, ``inst`` [W, H] int32
    raw ids (instance + 1, dataset.py:247) and ``cls`` [W, H] int32 classes (both None in iMAP mode), and ``T`` the
    GT camera-to-world pose [4, 4] fp64, which may hold non-finite entries.  Tensors are on the host."""
    if cfg.dataset_format != "ScanNet":
        raise ValueError(f"vmap_b200.scannet.read_sequence reads ScanNet configs, not {cfg.dataset_format}")
    ds = ScanNet(cfg, n_trackers=0)
    frames = list(range(len(ds))) if frames is None else list(frames)

    def load(i):
        color, depth, T, inst, sem = ds.decode_at(i)
        out = {"index": i, "rgb": torch.from_numpy(np.ascontiguousarray(color.transpose(1, 0, 2))),
               "depth": torch.from_numpy(np.ascontiguousarray(depth.T)), "T": np.asarray(T, np.float64),
               "inst": None, "cls": None}
        if inst is not None:
            out["inst"] = torch.from_numpy(np.ascontiguousarray(inst.T))
            semc = np.clip(sem.astype(np.int64), -1, None).astype(np.int32)      # as ScanNet.associate passes it
            out["cls"] = torch.from_numpy(np.ascontiguousarray(semc.T))
        return out

    with ThreadPoolExecutor(max_workers=max(prefetch, 1)) as pool:
        futs = {}
        for j in range(min(prefetch, len(frames))):
            futs[j] = pool.submit(load, frames[j])
        for j in range(len(frames)):
            nxt = j + prefetch
            if nxt < len(frames):
                futs[nxt] = pool.submit(load, frames[nxt])
            yield futs.pop(j).result() if j in futs else load(frames[j])


_BOX_FILTER_TRACKERS = {}


def box_filter(masks, classes, depth, inst_dict, intrinsic_open3d, T_CW, min_pixels=500, voxel_size=0.01):
    """utils.box_filter's signature and return value (int64 [H, W] numpy) over the GPU tracker.  The tracking
    state lives with ``inst_dict`` (one tracker per dict object), which receives ``InstData`` entries."""
    entry = _BOX_FILTER_TRACKERS.get(id(inst_dict))
    depth = np.asarray(depth, np.float32)
    Hh, Ww = depth.shape
    if entry is None or entry[0] is not inst_dict:
        if hasattr(intrinsic_open3d, "intrinsic_matrix"):
            K = np.asarray(intrinsic_open3d.intrinsic_matrix)
            fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
        else:
            fx, fy, cx, cy = intrinsic_open3d
        dev = torch.device("cuda", torch.cuda.current_device())
        entry = (inst_dict, InstanceTracker(fx, fy, cx, cy, dev, min_pixels, voxel_size, inst_dict=inst_dict))
        _BOX_FILTER_TRACKERS[id(inst_dict)] = entry
    tracker = entry[1]
    ids = np.zeros((Hh, Ww), np.int32)
    for m, c in zip(masks, classes):
        m = m.cpu().numpy() if torch.is_tensor(m) else np.asarray(m)
        if int(c) != 0:
            ids[m.astype(bool)] = int(c)
    labels, _ = tracker.frame(np.ascontiguousarray(ids.T), np.ascontiguousarray(depth.T),
                              camera_pose=np.linalg.inv(np.asarray(T_CW, np.float64)),
                              max_id=int(ids.max()) + 1, relabel=False)
    return labels.T.cpu().numpy()
