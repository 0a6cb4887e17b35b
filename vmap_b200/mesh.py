"""Meshing path of train.py's visualisation block (train.py:343-368): object bounds (sceneObject.get_bound,
vmap.py:270-315) and marching cubes (Trainer.meshing, trainer.py:35-75, vis.py:6-29).

Per-pixel and per-voxel arithmetic runs in the library: the object-pixel unprojection and marching cubes (K5,
csrc/k_mesh.cuh), the exact convex hull of the unprojected points and the minimum-volume box fitted to it (K8,
csrc/k_hull.cuh).  The host keeps the ``Mesh`` container that train.py exports, and ``oriented_bounds``, the host
restatement of trimesh's box fit that the device fit is checked against.  There is no CPU fallback: without the
library every device call raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, NamedTuple, Optional, Tuple, Union

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


# ---- exact convex hull and minimum-volume box on the device (K8) ----------------------------------------------------
class Hull(NamedTuple):
    """Convex hull of one point set: ``vertices`` int64 [V] indices of the extreme points in input order (scipy's
    ``ConvexHull.vertices`` order), ``facets`` int64 [F, 3] outward triangles (normal along (b - a) x (c - a)), both
    on the points' device; ``status`` one of _lib.HULL_OK / HULL_TOO_FEW (< 4 points) / HULL_FLAT (coplanar,
    collinear or identical points), with no vertices and no facets unless OK."""
    vertices: torch.Tensor
    facets: torch.Tensor
    status: int


def _as_points64(points, device=None) -> torch.Tensor:
    t = torch.as_tensor(points)
    if device is None:
        device = t.device if t.is_cuda else torch.device("cuda", torch.cuda.current_device())
    t = t.to(device=device, dtype=torch.float64).reshape(-1, 3).contiguous()
    return t


def _hull_launch(k: _Kernels, pts: torch.Tensor, sizes: torch.Tensor, stride: int, n_sets: int, nbr: bool = False):
    """Enqueues vmb_hull on fp64 points [n, 3] split into n_sets sets (set s has sizes[s * stride] points); returns
    the device outputs.  No host sync."""
    dev, n = pts.device, pts.shape[0]
    i32 = dict(dtype=torch.int32, device=dev)
    o = {"is_vertex": torch.empty(max(n, 1), dtype=torch.uint8, device=dev),
         "vertex_count": torch.empty(n_sets, **i32), "vertex_offset": torch.empty(n_sets + 1, **i32),
         "vertices": torch.empty(max(n, 1), **i32), "status": torch.empty(n_sets, **i32),
         "facets": torch.empty(max(2 * n, 1), 3, **i32), "facet_count": torch.empty(n_sets, **i32),
         "facet_nbr": torch.empty(max(2 * n, 1), 3, **i32) if nbr else None}
    a = _lib.HullArgs()
    a.points, a.n_points, a.set_size, a.size_stride, a.n_sets = _p(pts) if n else None, n, _p(sizes), stride, n_sets
    for f in ("is_vertex", "vertex_count", "vertex_offset", "vertices", "status", "facets", "facet_nbr",
              "facet_count"):
        setattr(a, f, _p(o[f]))
    k.call("vmb_hull", a)
    return o


def convex_hull(points: Union[torch.Tensor, np.ndarray, List]) -> Union[Hull, List[Hull]]:
    """Exact convex hull (K8) of one point set [n, 3], or of each set in a list (one launch for all).  Points are
    taken in fp64 (fp32 converts exactly) on their CUDA device, or the current one for host input.  A vertex is an
    extreme point: points on a facet or an edge are not vertices, and of several copies of an extreme point only the
    lowest index is one.  Returns a Hull per set, indices relative to that set."""
    single = torch.is_tensor(points) or isinstance(points, np.ndarray)
    sets = [points] if single else list(points)
    if not sets:
        return []
    first = torch.as_tensor(sets[0])
    dev = first.device if first.is_cuda else torch.device("cuda", torch.cuda.current_device())
    parts = [_as_points64(p, dev) for p in sets]
    pts = torch.cat(parts) if len(parts) > 1 else parts[0]
    counts = [int(p.shape[0]) for p in parts]
    sizes = torch.tensor(counts, dtype=torch.int32, device=dev)
    o = _hull_launch(_kernels(dev), pts, sizes, 1, len(parts))
    meta = torch.cat([o["vertex_offset"], o["status"], o["facet_count"]]).cpu().numpy()
    ns = len(parts)
    vo, st, fc = meta[:ns + 1], meta[ns + 1:2 * ns + 1], meta[2 * ns + 1:]
    out, start = [], 0
    for s, c in enumerate(counts):
        v = o["vertices"][int(vo[s]):int(vo[s + 1])].long() - start
        f = o["facets"][2 * start:2 * start + int(fc[s])].long() - start
        out.append(Hull(v, f, int(st[s])))
        start += c
    return out[0] if single else out


def oriented_bounds_gpu(points):
    """``oriented_bounds`` on the device: exact hull (K8), then the minimum-volume box over its distinct facet normals
    (vmb_obb_minvol), with no host round trip of the points; only the 15 numbers of the box come back.  Returns
    (center [3], R [3, 3] with the box axes as columns and det +1, extent [3]) as fp64 numpy.  Raises ValueError
    when the points are fewer than 4 or flat (coplanar, collinear or identical)."""
    pts = _as_points64(points)
    dev, n = pts.device, pts.shape[0]
    k = _kernels(dev)
    sizes = torch.tensor([n], dtype=torch.int32, device=dev)
    o = _hull_launch(k, pts, sizes, 1, 1, nbr=True)
    box = torch.empty(16, dtype=torch.float64, device=dev)
    status = torch.empty(1, dtype=torch.int32, device=dev)
    a = _lib.ObbArgs()
    a.points, a.facets, a.facet_nbr, a.facet_count = _p(pts) if n else _p(box), _p(o["facets"]), _p(o["facet_nbr"]), \
        _p(o["facet_count"])
    a.vertices, a.vertex_count, a.status = _p(o["vertices"]), _p(o["vertex_count"]), _p(o["status"])
    a.max_facets, a.box, a.box_status = max(2 * n, 1), _p(box), _p(status)
    k.call("vmb_obb_minvol", a)
    box[15] = status[0].to(torch.float64)
    b = box.cpu().numpy()
    st = int(b[15])
    if st != _lib.HULL_OK:
        raise ValueError("oriented_bounds_gpu: " + ("fewer than 4 points" if st == _lib.HULL_TOO_FEW else
                                                    "the points are flat (coplanar, collinear or identical)"))
    return b[0:3].copy(), b[3:12].reshape(3, 3).copy(), b[12:15].copy()
