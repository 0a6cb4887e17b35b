"""Meshing path of train.py's visualisation block (train.py:343-368): object bounds (sceneObject.get_bound,
vmap.py:270-315) and marching cubes (Trainer.meshing, trainer.py:35-75, vis.py:6-29).

Per-pixel and per-voxel arithmetic runs in the library (K5, csrc/k_mesh.cuh): the object-pixel unprojection and
marching cubes.  The host keeps what is small and sequential: the convex hull of the unprojected points
(scipy.spatial.ConvexHull) and the minimum-volume box fitted to it, and the ``Mesh`` container that train.py
exports.  There is no CPU fallback: without the library every call raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class _Kernels:
    """A library handle per device; owns the grow-only meshing scratch."""

    def __init__(self, device: torch.device):
        self.device, self.lib = device, _lib.lib()
        self._handle = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(None, self.lib.vmb_create(C.byref(self._handle), device.index or 0, 1, 32, 6), "vmb_create")

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self.lib.vmb_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def call(self, name, args):
        with torch.cuda.device(self.device):
            _lib.check(self._handle, getattr(self.lib, name)(
                self._handle, C.byref(args), C.c_void_p(torch.cuda.current_stream().cuda_stream)), name)


_KERNELS: Dict[str, _Kernels] = {}


def _kernels(device) -> _Kernels:
    device = torch.device(device)
    if device.type != "cuda":
        raise _lib.VmbError("meshing runs on a CUDA device: there is no CPU fallback")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    key = str(device)
    if key not in _KERNELS:
        _KERNELS[key] = _Kernels(device)
    return _KERNELS[key]


# ---- marching cubes -------------------------------------------------------------------------------------------------
def marching_cubes(volume: torch.Tensor, level: float = 0.5, affine=None):
    """(vertices [V,3] f32, faces [F,3] int32, normals [V,3] f32) on the volume's device, or None when the level is
    not crossed.  ``volume`` [nx,ny,nz]; ``affine`` [3,4] index -> world (identity by default).  Order and arithmetic
    are those of oracle/mesh_oracle.marching_cubes.  One host sync (to size the outputs)."""
    assert volume.dim() == 3 and volume.is_cuda
    vol = volume.to(torch.float32).contiguous()
    k = _kernels(vol.device)
    a = _lib.McArgs()
    a.volume, (a.nx, a.ny, a.nz), a.level = _p(vol), tuple(vol.shape), float(level)
    A = np.hstack([np.eye(3), np.zeros((3, 1))]) if affine is None else np.asarray(affine, dtype=np.float64)
    assert A.shape == (3, 4)
    a.affine[:] = [float(x) for x in A.reshape(-1)]
    totals = torch.zeros(2, dtype=torch.int32, device=vol.device)
    a.totals = _p(totals)
    k.call("vmb_mc_count", a)
    nv, nf = totals.tolist()
    if nv == 0 or nf == 0:
        return None
    verts = torch.empty(nv, 3, dtype=torch.float32, device=vol.device)
    normals = torch.empty_like(verts)
    faces = torch.empty(nf, 3, dtype=torch.int32, device=vol.device)
    a.vertices, a.normals, a.faces, a.max_vertices, a.max_faces = _p(verts), _p(normals), _p(faces), nv, nf
    k.call("vmb_mc_emit", a)
    return verts, faces, normals


class _Visual:
    def __init__(self, vertex_colors):
        self.vertex_colors = vertex_colors


class Mesh:
    """What train.py:360-364 and vis.py:21-29 use of a trimesh.Trimesh: ``vertices``, ``faces``, ``vertex_normals``,
    ``visual.vertex_colors`` (N x 4 RGBA uint8) and ``export(path)`` to Wavefront .obj."""

    def __init__(self, vertices, faces, vertex_normals, vertex_colors):
        self.vertices = np.asarray(vertices)
        self.faces = np.asarray(faces)
        self.vertex_normals = np.asarray(vertex_normals)
        self.visual = _Visual(np.asarray(vertex_colors, dtype=np.uint8))

    def export(self, path: str) -> None:
        """Wavefront .obj: ``v x y z r g b`` (colour in [0, 1]), ``vn``, 1-based ``f a//a b//b c//c``."""
        if os.path.splitext(path)[1].lower() != ".obj":
            raise ValueError("Mesh.export writes .obj only")
        v = np.asarray(self.vertices, np.float64)
        c = self.visual.vertex_colors[:, :3].astype(np.float64) / 255.0
        f = np.asarray(self.faces, np.int64) + 1
        with open(path, "w") as fh:
            fh.write(f"# {len(v)} vertices, {len(f)} faces\n")
            fh.write("".join(f"v {x:.8g} {y:.8g} {z:.8g} {r:.6g} {g:.6g} {b:.6g}\n"
                             for (x, y, z), (r, g, b) in zip(v.tolist(), c.tolist())))
            fh.write("".join(f"vn {x:.8g} {y:.8g} {z:.8g}\n" for x, y, z in np.asarray(self.vertex_normals).tolist()))
            fh.write("".join(f"f {a}//{a} {b}//{b} {d}//{d}\n" for a, b, d in f.tolist()))


# ---- object bounds --------------------------------------------------------------------------------------------------
def intrinsic_matrix(intrinsic) -> np.ndarray:
    """3x3 K from an open3d PinholeCameraIntrinsic (``.intrinsic_matrix``) or anything array-like."""
    K = np.asarray(getattr(intrinsic, "intrinsic_matrix", intrinsic), dtype=np.float64)
    if K.shape != (3, 3):
        raise ValueError(f"intrinsic matrix must be 3x3, got {K.shape}")
    return K


def unproject_object(obj, K: np.ndarray) -> torch.Tensor:
    """World points [n,3] f32 (on the object's data device) of every pixel of the object's keyframes that belongs to
    it and has depth > 0 (vmap.py:272-286), in (keyframe, u, v) order."""
    dev = torch.device(obj.data_device)
    k = _kernels(dev)
    a = _lib.UnprojectArgs()
    a.width, a.height, a.n_keyframes = obj.frames_width, obj.frames_height, int(obj.n_keyframes)
    a.fx, a.fy, a.cx, a.cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    if obj.store is not None:
        st = obj.store
        slots = torch.tensor(obj.kf_store_slot[:obj.n_keyframes], dtype=torch.int32, device=dev)
        a.store_depth, a.store_inst, a.store_t_wc, a.kf_slot = _p(st.depth), _p(st.inst), _p(st.t_wc), _p(slots)
        a.obj_id = int(obj.obj_id)
    else:
        for t in (obj.rgbs_batch, obj.depth_batch, obj.t_wc_batch):
            assert t.is_contiguous() and t.device == dev
        a.rgbs, a.depths, a.t_wc = _p(obj.rgbs_batch), _p(obj.depth_batch), _p(obj.t_wc_batch)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    a.count = _p(count)
    k.call("vmb_unproject", a)
    n = int(count.item())
    pts = torch.empty(n, 3, dtype=torch.float32, device=dev)
    if n:
        a.points, a.max_points = _p(pts), n
        k.call("vmb_unproject", a)
    return pts


def _min_area_rect(p2: np.ndarray) -> Tuple[float, np.ndarray, np.ndarray, np.ndarray]:
    """Rotating calipers over the edges of the 2-D convex hull of ``p2``: (area, unit edge direction, lo, hi) of the
    minimum-area enclosing rectangle, lo / hi its bounds along (direction, perpendicular)."""
    from scipy.spatial import ConvexHull
    h = p2[ConvexHull(p2).vertices]
    e = np.roll(h, -1, axis=0) - h
    ln = np.linalg.norm(e, axis=1)
    d = e[ln > 0] / ln[ln > 0, None]
    u = h @ d.T                                              # [P, E] along each edge
    w = h @ np.stack([-d[:, 1], d[:, 0]], 1).T               # [P, E] perpendicular
    area = (u.max(0) - u.min(0)) * (w.max(0) - w.min(0))
    i = int(np.argmin(area))
    return float(area[i]), d[i], np.array([u[:, i].min(), w[:, i].min()]), np.array([u[:, i].max(), w[:, i].max()])


def oriented_bounds(points: np.ndarray):
    """Minimum-volume oriented box of a point set, trimesh.bounds.oriented_bounds' algorithm restated: for every
    distinct face normal of the convex hull, project the hull onto the plane normal to it, take the minimum-area
    rectangle of the projection (rotating calipers) and keep the box of least volume.  Returns (center [3],
    R [3,3] with the box axes as columns and det +1, extent [3]).  Raises scipy's QhullError when the points are
    too few or degenerate (coplanar)."""
    from scipy.spatial import ConvexHull
    pts = np.asarray(points, dtype=np.float64)
    hull = ConvexHull(pts)
    hv = pts[hull.vertices]
    normals = hull.equations[:, :3]
    normals = normals / np.linalg.norm(normals, axis=1, keepdims=True)
    normals = np.unique(np.round(normals, 10), axis=0)
    best = None
    for n in normals:
        b1 = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0])
        b1 /= np.linalg.norm(b1)
        b2 = np.cross(n, b1)
        h = hv @ n
        height = h.max() - h.min()
        try:
            area, d, lo, hi = _min_area_rect(np.stack([hv @ b1, hv @ b2], 1))
        except Exception:                                    # degenerate projection (cannot happen for a 3-D hull)
            continue
        vol = area * height
        if best is None or vol < best[0]:
            a0 = d[0] * b1 + d[1] * b2
            a1 = -d[1] * b1 + d[0] * b2
            R = np.stack([a0, a1, n], 1)
            mid = np.array([(lo[0] + hi[0]) / 2, (lo[1] + hi[1]) / 2, (h.max() + h.min()) / 2])
            ext = np.array([hi[0] - lo[0], hi[1] - lo[1], height])
            best = (vol, R, mid, ext)
    _, R, mid, ext = best
    if np.linalg.det(R) < 0:                                 # proper rotation: flip the normal axis
        R[:, 2] = -R[:, 2]
        mid[2] = -mid[2]
    return R @ mid, R, ext
