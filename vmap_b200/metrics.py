"""3-D reconstruction metrics of the vMAP paper (metric/metrics.py, eval_3D_obj.py, eval_3D_scene.py) on the GPU.

``accuracy`` / ``completion`` / ``completion_ratio`` / ``chamfer`` keep metric/metrics.py's names, argument order and
meaning; ``calc_3d_metric`` is eval_3D_scene.calc_3d_metric, and with ``crop_to_gt_box=True`` eval_3D_obj's variant.
Surface sampling, the box crop and the exact nearest-neighbour distances run in the library (K6, csrc/k_eval.cuh);
means and ratios are fp64 torch reductions over the kernel's per-point fp32 distances.  There is no CPU fallback:
without the library or a CUDA device every GPU call raises.

Meshes are a ``vmap_b200.mesh.Mesh``, anything with ``.vertices`` / ``.faces`` (a trimesh object works), or a
``(vertices, faces)`` pair.  ``load_mesh`` reads .obj and .ply (ascii and binary_little_endian) without trimesh.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .mesh import _kernels, _p, oriented_bounds_gpu

# the reference's background classes (eval_3D_obj.py:68)
BACKGROUND_CLS = [5, 12, 30, 31, 40, 60, 92, 93, 95, 97, 98, 79]
# the ground-truth samples are drawn from another Philox key than the reconstruction's
_GT_SEED_XOR = 0x9E3779B97F4A7C15


class TriangleMesh:
    """An indexed triangle mesh as read from disk: ``vertices`` [V,3] float64, ``faces`` [F,3] int64."""

    def __init__(self, vertices, faces):
        self.vertices = np.asarray(vertices, np.float64).reshape(-1, 3)
        self.faces = np.asarray(faces, np.int64).reshape(-1, 3)


def _device(device=None) -> torch.device:
    if device is None:
        if not torch.cuda.is_available():
            raise _lib.VmbError("the evaluation metrics run on a CUDA device: there is no CPU fallback")
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device(device)


def _points(x, device) -> torch.Tensor:
    t = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
    t = t.to(device=device, dtype=torch.float32).reshape(-1, 3).contiguous()
    return t


def _mesh_tensors(mesh, device) -> Tuple[torch.Tensor, torch.Tensor]:
    if isinstance(mesh, (tuple, list)) and len(mesh) == 2:
        v, f = mesh
    else:
        v, f = mesh.vertices, mesh.faces
    f = torch.as_tensor(np.asarray(f) if not torch.is_tensor(f) else f)
    return _points(v, device), f.to(device=device, dtype=torch.int32).reshape(-1, 3).contiguous()


# ---- kernels --------------------------------------------------------------------------------------------------------
def nn_dist(ref, query, with_index: bool = False, device=None):
    """Exact nearest-neighbour distance [n_q] f32 (and index [n_q] int32, ties to the lowest ref index) of every query
    point to the ref set, on the GPU."""
    dev = _device(device if device is not None else (ref.device if torch.is_tensor(ref) and ref.is_cuda else None))
    r, q = _points(ref, dev), _points(query, dev)
    dist = torch.empty(q.shape[0], dtype=torch.float32, device=dev)
    index = torch.empty(q.shape[0], dtype=torch.int32, device=dev) if with_index else None
    a = _lib.NnArgs()
    a.ref, a.n_ref, a.query, a.n_query, a.dist, a.index = _p(r), r.shape[0], _p(q), q.shape[0], _p(dist), _p(index)
    _kernels(dev).call("vmb_nn_dist", a)
    return (dist, index) if with_index else dist


def sample_surface(mesh, count: int, seed: int = 0, uniforms=None, device=None):
    """(points [count,3] f32, face_index [count] int32) on the GPU: trimesh.sample.sample_surface's area-weighted rule
    with Philox randoms keyed by ``seed``; ``uniforms`` [count,3] (u0, u1, u2) replaces them."""
    dev = _device(device)
    v, f = _mesh_tensors(mesh, dev)
    pts = torch.empty(int(count), 3, dtype=torch.float32, device=dev)
    fi = torch.empty(int(count), dtype=torch.int32, device=dev)
    u = None
    if uniforms is not None:
        u = torch.as_tensor(np.asarray(uniforms) if not torch.is_tensor(uniforms) else uniforms)
        u = u.to(device=dev, dtype=torch.float64).contiguous()
        assert u.shape == (int(count), 3)
    a = _lib.SurfaceSampleArgs()
    a.vertices, a.n_vertices, a.faces, a.n_faces = _p(v), v.shape[0], _p(f), f.shape[0]
    a.n_points, a.seed, a.uniforms, a.points, a.face_index = int(count), int(seed) & (2 ** 64 - 1), _p(u), _p(pts), _p(fi)
    _kernels(dev).call("vmb_surface_sample", a)
    return pts, fi


def crop_to_box(mesh, center, R, extent, device=None) -> Optional[torch.Tensor]:
    """mesh ∩ box as a triangle soup [T,3,3] f32 on the GPU, ordered by (input face, fan order), or None when nothing is
    left.  ``R`` has the box axes as columns, ``extent`` the full edge lengths.  One host sync."""
    dev = _device(device)
    v, f = _mesh_tensors(mesh, dev)
    k = _kernels(dev)
    a = _lib.ClipArgs()
    a.vertices, a.n_vertices, a.faces, a.n_faces = _p(v), v.shape[0], _p(f), f.shape[0]
    a.center[:] = [float(x) for x in np.asarray(center, np.float64).reshape(3)]
    a.rotation[:] = [float(x) for x in np.asarray(R, np.float64).reshape(9)]
    a.extent[:] = [float(x) for x in np.asarray(extent, np.float64).reshape(3)]
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    a.count = _p(count)
    k.call("vmb_clip_count", a)
    T = int(count.item())
    if T == 0:
        return None
    soup = torch.empty(T, 3, 3, dtype=torch.float32, device=dev)
    a.triangles, a.max_triangles = _p(soup), T
    k.call("vmb_clip_emit", a)
    return soup


def soup_mesh(soup: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """A triangle soup as an indexed mesh: (vertices [3T,3], faces = arange(3T).view(T,3))."""
    T = soup.shape[0]
    return soup.reshape(-1, 3), torch.arange(3 * T, dtype=torch.int32, device=soup.device).view(T, 3)


# ---- metric/metrics.py ----------------------------------------------------------------------------------------------
def _dev_of(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    return _device()


def accuracy(gt_points, rec_points) -> float:
    """Mean over the reconstruction's points of the distance to the nearest ground-truth point."""
    return float(nn_dist(gt_points, rec_points, device=_dev_of(gt_points, rec_points)).double().mean())


def completion(gt_points, rec_points) -> float:
    """Mean over the ground-truth points of the distance to the nearest reconstructed point."""
    return float(nn_dist(rec_points, gt_points, device=_dev_of(gt_points, rec_points)).double().mean())


def completion_ratio(gt_points, rec_points, dist_th=0.01) -> float:
    """Fraction of the ground-truth points whose nearest reconstructed point is closer than ``dist_th``."""
    d = nn_dist(rec_points, gt_points, device=_dev_of(gt_points, rec_points))
    return _ratio(d, dist_th)


def _ratio(d: torch.Tensor, th: float) -> float:
    """Fraction of d below th as the correctly rounded count / n (what numpy's mean of 0 / 1 values gives)."""
    return int((d < th).sum()) / d.numel() if d.numel() else float("nan")


def chamfer(gt_points, rec_points) -> float:
    return (completion(gt_points, rec_points) + accuracy(gt_points, rec_points)) / 2.0


# ---- eval_3D_*.calc_3d_metric ---------------------------------------------------------------------------------------
def calc_3d_metric(mesh_rec, mesh_gt, N: int = 200000, crop_to_gt_box: bool = False, seed: int = 0, uniforms=None,
                   device=None):
    """[[accuracy], [completion], [completion ratio @ 1 cm], [completion ratio @ 5 cm]] of a reconstruction against
    its ground truth, N surface samples each.  ``crop_to_gt_box`` first cuts the reconstruction to the ground truth's
    minimum-volume oriented box enlarged by 1 / 0.9 (eval_3D_obj.py) and returns None when nothing is left.
    ``uniforms`` = (rec [N,3], gt [N,3]) replaces the Philox randoms (to reproduce another implementation's samples).
    One nearest-neighbour query per direction: completion and both ratios share the gt -> rec distances."""
    dev = _device(device)
    if crop_to_gt_box:
        gt_v = mesh_gt[0] if isinstance(mesh_gt, (tuple, list)) else mesh_gt.vertices
        gt_v = gt_v.detach() if torch.is_tensor(gt_v) else torch.from_numpy(np.asarray(gt_v, np.float64))
        center, R, ext = oriented_bounds_gpu(gt_v.to(dev))
        soup = crop_to_box(mesh_rec, center, R, ext / 0.9, device=dev)
        if soup is None:
            print("no mesh found")
            return None
        mesh_rec = soup_mesh(soup)
    u_rec, u_gt = (None, None) if uniforms is None else uniforms
    rec, _ = sample_surface(mesh_rec, N, seed=seed, uniforms=u_rec, device=dev)
    gt, _ = sample_surface(mesh_gt, N, seed=seed ^ _GT_SEED_XOR, uniforms=u_gt, device=dev)
    d_rec = nn_dist(gt, rec, device=dev).double()             # rec -> gt: accuracy
    d_gt = nn_dist(rec, gt, device=dev).double()              # gt -> rec: completion and its ratios
    return [[float(d_rec.mean())], [float(d_gt.mean())], [_ratio(d_gt, 0.01)], [_ratio(d_gt, 0.05)]]


# ---- loading --------------------------------------------------------------------------------------------------------
def _fan(poly: Sequence[int]) -> List[List[int]]:
    return [[poly[0], poly[k], poly[k + 1]] for k in range(1, len(poly) - 1)]


def _load_obj(path) -> TriangleMesh:
    v, f = [], []
    with open(path) as fh:
        for line in fh:
            t = line.split()
            if not t:
                continue
            if t[0] == "v":
                v.append([float(x) for x in t[1:4]])
            elif t[0] == "f":
                idx = [int(x.split("/")[0]) for x in t[1:]]
                idx = [i - 1 if i > 0 else len(v) + i for i in idx]          # 1-based, negative = relative
                f.extend(_fan(idx))
    return TriangleMesh(np.asarray(v, np.float64).reshape(-1, 3), np.asarray(f, np.int64).reshape(-1, 3))


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _ply_header(fh):
    if fh.readline().strip() != b"ply":
        raise ValueError("not a PLY file")
    fmt, elements = None, []
    while True:
        line = fh.readline()
        if not line:
            raise ValueError("PLY header without end_header")
        t = line.decode("ascii", "replace").split()
        if not t or t[0] in ("comment", "obj_info"):
            continue
        if t[0] == "format":
            fmt = t[1]
        elif t[0] == "element":
            elements.append((t[1], int(t[2]), []))
        elif t[0] == "property":
            if t[1] == "list":                                   # property list <count type> <item type> <name>
                elements[-1][2].append((t[4], _PLY_TYPES[t[2]], _PLY_TYPES[t[3]]))
            else:
                elements[-1][2].append((t[2], _PLY_TYPES[t[1]], None))
        elif t[0] == "end_header":
            return fmt, elements


def _ply_binary_element(buf, pos, count, props):
    """(columns {name: array or list of lists}, new position) of one binary little-endian element."""
    if all(p[2] is None for p in props):
        dt = np.dtype([(n, "<" + t) for n, t, _ in props])
        a = np.frombuffer(buf, dt, count, pos)
        return {n: a[n] for n, _, _ in props}, pos + count * dt.itemsize
    if count == 0:
        return {n: [] for n, _, _ in props}, pos
    # guess that every list has the length of the first one, check, and fall back to a per-element walk
    fields, off = [], pos
    for n, t, it in props:
        if it is None:
            fields.append((n, "<" + t)); off += np.dtype(t).itemsize
        else:
            k = int(np.frombuffer(buf, "<" + t, 1, off)[0])
            fields.append((n + "#n", "<" + t)); fields.append((n, "<" + it, (k,)))
            off += np.dtype(t).itemsize + k * np.dtype(it).itemsize
    dt = np.dtype(fields)
    if pos + count * dt.itemsize <= len(buf):
        a = np.frombuffer(buf, dt, count, pos)
        if all((a[n + "#n"] == a.dtype[n].shape[0]).all() for n, _, it in props if it is not None):
            return {n: a[n] for n, _, _ in props}, pos + count * dt.itemsize
    cols = {n: [] for n, _, _ in props}
    for _ in range(count):
        for n, t, it in props:
            if it is None:
                cols[n].append(np.frombuffer(buf, "<" + t, 1, pos)[0]); pos += np.dtype(t).itemsize
            else:
                k = int(np.frombuffer(buf, "<" + t, 1, pos)[0]); pos += np.dtype(t).itemsize
                cols[n].append(np.frombuffer(buf, "<" + it, k, pos).tolist()); pos += k * np.dtype(it).itemsize
    return cols, pos


def _load_ply(path) -> TriangleMesh:
    with open(path, "rb") as fh:
        fmt, elements = _ply_header(fh)
        body = fh.read()
    data = {}
    if fmt == "binary_little_endian":
        pos = 0
        for name, count, props in elements:
            data[name], pos = _ply_binary_element(body, pos, count, props)
    elif fmt == "ascii":
        lines = iter(body.decode("ascii").split("\n"))
        for name, count, props in elements:
            cols = {n: [] for n, _, _ in props}
            for _ in range(count):
                t = next(lines).split()
                while not t:
                    t = next(lines).split()
                i = 0
                for n, _, it in props:
                    if it is None:
                        cols[n].append(float(t[i])); i += 1
                    else:
                        k = int(t[i]); cols[n].append([int(float(x)) for x in t[i + 1:i + 1 + k]]); i += 1 + k
            data[name] = cols
    else:
        raise ValueError(f"unsupported PLY format {fmt!r} (ascii and binary_little_endian are read)")
    vx = data.get("vertex", {})
    v = np.stack([np.asarray(vx[c], np.float64) for c in ("x", "y", "z")], 1) if vx else np.zeros((0, 3))
    fc = data.get("face", {})
    key = "vertex_indices" if "vertex_indices" in fc else ("vertex_index" if "vertex_index" in fc else None)
    if key is None:
        return TriangleMesh(v, np.zeros((0, 3), np.int64))
    lists = fc[key]
    if isinstance(lists, np.ndarray):                              # every face has the same number of corners
        L = lists.astype(np.int64)
        f = np.concatenate([L[:, [0, k, k + 1]] for k in range(1, L.shape[1] - 1)], 1).reshape(-1, 3) \
            if L.shape[1] >= 3 else np.zeros((0, 3), np.int64)
    else:
        f = [tri for poly in lists for tri in _fan(list(poly))]
    return TriangleMesh(v, np.asarray(f, np.int64).reshape(-1, 3))


def load_mesh(path) -> TriangleMesh:
    """Vertices and triangles of a .obj (``v`` / ``f`` lines, ``f a``, ``a//n``, ``a/t/n`` forms) or .ply (ascii or
    binary_little_endian; x, y, z as float or double; every other property skipped by its declared type).  Polygons
    are fan-triangulated from their first corner."""
    ext = os.path.splitext(str(path))[1].lower()
    if ext == ".obj":
        return _load_obj(path)
    if ext == ".ply":
        return _load_ply(path)
    raise ValueError(f"load_mesh reads .obj and .ply, not {ext!r}")


def concatenate(meshes) -> TriangleMesh:
    """One mesh of several (trimesh.util.concatenate): vertices stacked, face indices offset."""
    vs, fs, off = [], [], 0
    for m in meshes:
        v = np.asarray(m[0] if isinstance(m, (tuple, list)) else m.vertices, np.float64).reshape(-1, 3)
        f = np.asarray(m[1] if isinstance(m, (tuple, list)) else m.faces, np.int64).reshape(-1, 3)
        vs.append(v); fs.append(f + off); off += len(v)
    if not vs:
        return TriangleMesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64))
    return TriangleMesh(np.concatenate(vs), np.concatenate(fs))


def frame_obj_ids(mesh_dir, frame: int) -> List[int]:
    """Object ids of the ``frame_{frame}_obj{id}.obj`` files train.py wrote into ``mesh_dir``, ascending."""
    pat = re.compile(r"^frame_%d_obj(\d+)\.obj$" % int(frame))
    return sorted(int(m.group(1)) for m in (pat.match(f) for f in os.listdir(mesh_dir)) if m)


def view_metrics(colour, depth, gt_rgb, gt_depth, gt_inst=None) -> dict:
    """2-D view metrics of a rendered view (vmap_b200.render.render_view) against ground truth, all images [W, H, ...].
    The reference never published its eval_2D_view.py, so these definitions are the package's own:
      psnr      over all pixels, colours in [0, 1], MSE in fp64;
      depth_l1  mean |depth - gt| in metres over pixels with gt > 0 (nan when there are none);
      obj_psnr  (with ``gt_inst``) the mean over GT instances != 0 of each instance's PSNR over its pixels."""
    c = torch.as_tensor(colour).double()
    g = torch.as_tensor(gt_rgb).double().to(c.device)
    d = torch.as_tensor(depth).double().to(c.device)
    gd = torch.as_tensor(gt_depth).double().to(c.device)

    def psnr(mse):
        return float(-10.0 * torch.log10(mse)) if float(mse) > 0 else float("inf")

    se = ((c - g) ** 2).mean(-1)
    out = {"psnr": psnr(se.mean())}
    valid = gd > 0
    out["depth_l1"] = float((d - gd).abs()[valid].mean()) if bool(valid.any()) else float("nan")
    if gt_inst is not None:
        gi = torch.as_tensor(gt_inst).to(c.device)
        ids = [int(i) for i in torch.unique(gi).tolist() if int(i) != 0]
        vals = [psnr(se[gi == i].mean()) for i in ids]
        out["obj_psnr"] = float(np.mean(vals)) if vals else float("nan")
    return out


# ---- trajectory metrics (TUM RGB-D benchmark definitions; host fp64, N <= a few thousand poses once per run) ---------

def _poses(x) -> np.ndarray:
    a = np.asarray(x.detach().cpu() if torch.is_tensor(x) else x, np.float64)
    if a.ndim != 3 or a.shape[1:] != (4, 4):
        raise ValueError(f"expected camera-to-world poses [N, 4, 4], got {a.shape}")
    return a


def _positions(x) -> np.ndarray:
    a = np.asarray(x.detach().cpu() if torch.is_tensor(x) else x, np.float64)
    if a.ndim == 3 and a.shape[1:] == (4, 4):
        return a[:, :3, 3]
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError(f"expected poses [N, 4, 4] or positions [N, 3], got {a.shape}")
    return a


def align_se3(est, gt) -> np.ndarray:
    """The rigid transform S [4, 4] (rotation and translation, no scale) minimising sum_i |gt_i - S est_i|^2 over the
    positions (poses [N, 4, 4] or positions [N, 3]), in closed form (Umeyama 1991, "Least-squares estimation of
    transformation parameters between two point patterns", eqs. 38-42 with c = 1): with the centred cross-covariance
    Sigma = 1/N sum (gt_i - mu_gt)(est_i - mu_est)^T = U D V^T, R = U diag(1, 1, s) V^T where s = -1 when
    det(U) det(V) < 0 (the reflection guard) and 1 otherwise, and t = mu_gt - R mu_est.  The TUM benchmark's ATE uses
    the same alignment (Horn's method)."""
    e, g = _positions(est), _positions(gt)
    if e.shape != g.shape or len(e) < 1:
        raise ValueError("align_se3: est and gt need the same, non-zero number of poses")
    me, mg = e.mean(0), g.mean(0)
    sigma = (g - mg).T @ (e - me) / len(e)
    U, _, Vt = np.linalg.svd(sigma)
    s = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        s[2, 2] = -1.0
    S = np.eye(4)
    S[:3, :3] = U @ s @ Vt
    S[:3, 3] = mg - S[:3, :3] @ me
    return S


def _valid(valid, gt: np.ndarray) -> np.ndarray:
    """The frames a metric keeps: ``valid`` [N] (bool) and a GT pose (or position) with every entry finite."""
    v = np.asarray(valid, bool).reshape(-1)
    if v.shape[0] != len(gt):
        raise ValueError(f"valid needs one flag per frame ({len(gt)}), got {v.shape[0]}")
    return v & np.isfinite(gt.reshape(len(gt), -1)).all(1)


def ate(est, gt, align: bool = True, valid=None) -> dict:
    """Absolute trajectory error (Sturm et al. 2012, the TUM RGB-D benchmark, eq. 2): F_i = Q_i^-1 S P_i with P the
    estimate, Q the ground truth and S = ``align_se3(P, Q)`` (identity with ``align=False``); the residual of frame i
    is |trans(F_i)| = |q_i - S p_i| in metres.  Returns rmse, mean, median and max of the residuals (floats) and the
    per-frame ``errors`` [N] (numpy).  ``valid`` (optional [N] bool, e.g. all True): score only the frames it flags
    whose GT pose has no non-finite entry (ScanNet marks frames without a GT pose with inf); the result is the metric
    of that subset, and ``errors`` holds its frames only."""
    if valid is not None:
        g = np.asarray(gt.detach().cpu() if torch.is_tensor(gt) else gt, np.float64)
        e = np.asarray(est.detach().cpu() if torch.is_tensor(est) else est, np.float64)
        m = _valid(valid, g)
        if not m.any():
            raise ValueError("ate: no frame with a valid GT pose")
        return ate(e[m], g[m], align=align)
    e, g = _positions(est), _positions(gt)
    S = align_se3(e, g) if align else np.eye(4)
    err = np.linalg.norm(g - (e @ S[:3, :3].T + S[:3, 3]), axis=1)
    return {"rmse": float(np.sqrt(np.mean(err ** 2))), "mean": float(err.mean()), "median": float(np.median(err)),
            "max": float(err.max()), "errors": err}


def _inv_se3(T: np.ndarray) -> np.ndarray:
    inv = np.zeros_like(T)
    inv[:, :3, :3] = T[:, :3, :3].transpose(0, 2, 1)
    inv[:, :3, 3] = -np.einsum("nji,nj->ni", T[:, :3, :3], T[:, :3, 3])
    inv[:, 3, 3] = 1.0
    return inv


def _rel(T: np.ndarray, delta: int) -> np.ndarray:
    return _inv_se3(T[:-delta]) @ T[delta:]


def rpe(est, gt, delta: int = 1, valid=None) -> dict:
    """Relative pose error (Sturm et al. 2012, eq. 1) over ``delta`` frames: E_i = (Q_i^-1 Q_{i+d})^-1 (P_i^-1 P_{i+d}).
    Returns ``trans_rmse`` (metres), the RMSE of |trans(E_i)|, and ``rot_rmse_deg``, the RMSE of the rotation angle
    arccos((trace(rot(E_i)) - 1) / 2) in degrees, plus the per-pair ``trans_errors`` / ``rot_errors_deg``.  ``valid``
    (optional [N] bool): keep only the pairs (i, i + d) whose two frames it flags and whose two GT poses have no
    non-finite entry, as ``ate`` does per frame."""
    P, Q = _poses(est), _poses(gt)
    if P.shape != Q.shape or not 1 <= delta < len(P):
        raise ValueError("rpe: est and gt need the same number of poses, more than delta")
    if valid is not None:
        m = _valid(valid, Q)
        i = np.nonzero(m[:-delta] & m[delta:])[0]
        if len(i) == 0:
            raise ValueError("rpe: no pair of frames with valid GT poses")
        E = _inv_se3(_inv_se3(Q[i]) @ Q[i + delta]) @ (_inv_se3(P[i]) @ P[i + delta])
    else:
        E = _inv_se3(_rel(Q, delta)) @ _rel(P, delta)
    te = np.linalg.norm(E[:, :3, 3], axis=1)
    c = np.clip((np.trace(E[:, :3, :3], axis1=1, axis2=2) - 1.0) / 2.0, -1.0, 1.0)
    re = np.degrees(np.arccos(c))
    return {"trans_rmse": float(np.sqrt(np.mean(te ** 2))), "rot_rmse_deg": float(np.sqrt(np.mean(re ** 2))),
            "trans_errors": te, "rot_errors_deg": re}
