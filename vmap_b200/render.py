"""Render the object map from any camera on the GPU (K9): composited depth, colour, opacity and instance images.

Every object network is a *source* with an oriented box (the box ``Trainer.meshing`` evaluates in).  Rays are culled
against the boxes, sampled inside each hit box (coarse pass), composited front to back over all objects, then sampled
again in a band around the coarse surface (fine pass) and composited once more.  The rule -- ray convention, slab
test, sample positions, merge order and compositing -- is written down in ``csrc/k_render.cuh``;
``oracle/render_oracle.py`` restates it.  The network forward is ``VmapEnsemble.eval_points`` (``vmb_forward``) on each
source's contiguous segment of points.
"""
from __future__ import annotations

import ctypes as C
import warnings
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .ensemble import _ptr, _stream

MAX_HITS = _lib.RENDER_MAX_HITS


@dataclass
class Source:
    """One object network and its box: ``(ens, row)`` of the packed stack, the ``obj_id`` written into the instance
    image, box ``center`` [3], axes ``R`` [3,3] (columns) and ``half_extent`` [3]; ``offset`` is subtracted from
    world points before the network sees them (``obj_center``, 0 in the package)."""
    ens: object
    row: int
    obj_id: int
    center: Sequence[float]
    R: Sequence[Sequence[float]]
    half_extent: Sequence[float]
    offset: Sequence[float] = (0.0, 0.0, 0.0)


def sources_from_objects(objects) -> Tuple[List[Source], List[int]]:
    """Sources of drop-in ``sceneObject``s: ``(ens, row)`` from the module binding (as ``Trainer.eval_points``), the
    box from ``obj.bbox3d`` (set by ``get_bound``) with half-extents ``extent / (2 * trainer.bound_extent)``.
    Returns (sources, ids of the objects left out because they have no ``bbox3d``)."""
    from .lazy import ensemble_for_modules
    out, skipped = [], []
    for obj in objects:
        if obj.bbox3d is None:
            skipped.append(int(obj.obj_id))
            continue
        t = obj.trainer
        ens = ensemble_for_modules(t.fc_occ_map, t.pe)
        row = t.fc_occ_map._vmb_binding[1]
        b = obj.bbox3d
        half = np.asarray(b.extent, np.float64) / (2.0 * t.bound_extent)
        off = np.broadcast_to(np.asarray(torch.as_tensor(obj.obj_center).cpu(), np.float64), (3,))
        out.append(Source(ens, row, int(obj.obj_id), np.asarray(b.center, np.float64), np.asarray(b.R, np.float64),
                          half, off))
    return out, skipped


def box_table(sources: Sequence[Source]) -> np.ndarray:
    """[n_src, 18] fp64: center, R row-major, half extent, offset (the layout of vmb_render_args.boxes)."""
    t = np.zeros((len(sources), _lib.RENDER_BOX), np.float64)
    for i, s in enumerate(sources):
        t[i, 0:3] = np.asarray(s.center, np.float64).reshape(3)
        t[i, 3:12] = np.asarray(s.R, np.float64).reshape(9)
        t[i, 12:15] = np.asarray(s.half_extent, np.float64).reshape(3)
        t[i, 15:18] = np.asarray(s.offset, np.float64).reshape(3)
    return t


class _View:
    """One render call's fixed arguments (camera, sources, sample counts) in a vmb_render_args, and the C calls."""

    def __init__(self, sources, t_wc, K, width, height, n_coarse, n_fine, surface_eps, near, far):
        if not sources:
            raise _lib.VmbError("render_view: no sources")
        self.sources = list(sources)
        self.ens0 = self.sources[0].ens
        self.dev = self.ens0.device
        self.boxes = np.ascontiguousarray(box_table(self.sources))
        self.ids = np.ascontiguousarray([s.obj_id for s in self.sources], dtype=np.int32)
        T = np.asarray(torch.as_tensor(t_wc).double().cpu() if torch.is_tensor(t_wc) else t_wc, np.float64)
        K = np.asarray(K, np.float64)
        a = _lib.RenderArgs()
        a.width, a.height = int(width), int(height)
        a.fx, a.fy, a.cx, a.cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
        a.t_wc[:] = [float(x) for x in T[:3, :4].reshape(-1)]
        a.near_depth, a.far_depth, a.surface_eps = float(near), float(far), float(surface_eps)
        a.n_src = len(self.sources)
        a.boxes = C.c_void_p(self.boxes.ctypes.data)
        a.obj_id = C.c_void_p(self.ids.ctypes.data)
        a.n_coarse, a.n_fine = int(n_coarse), int(n_fine)
        self.a = a

    def call(self, fn: str, what: str):
        e = self.ens0
        with e._on_device():
            _lib.check(e._handle, getattr(e.lib, fn)(e._handle, C.byref(self.a), _stream()), what)


def _forward(sources, totals, points, alpha, colour, impl):
    """vmb_forward once per source row on that source's contiguous segment, straight into the pass's buffers."""
    off = 0
    for s, n in zip(sources, totals):
        if n > 0:
            s.ens.eval_points(points[off:off + n], impl=impl, row=s.row, out=(alpha[off:off + n], colour[off:off + n]))
        off += n


def render_view(sources: Sequence[Source], t_wc, K, width: int, height: int, n_coarse: int = 32, n_fine: int = 16,
                surface_eps: float = 0.1, near: float = 0.0, far: float = 1e4, chunk_rays: int = 1 << 17,
                impl=None, stages=None) -> Tuple[Dict[str, torch.Tensor], Dict[str, int]]:
    """Render a ``width`` x ``height`` view from camera-to-world pose ``t_wc`` [4,4] with intrinsics ``K`` [3,3].

    Returns ``images`` = {depth [W,H], colour [W,H,3], opacity [W,H], instance [W,H] int32 (obj ids, -1 = none),
    coarse_surface [W,H] int32 (index of the coarse pass's surface sample in the ray's merged sequence, -1 = none)} on
    the device, and ``stats`` = {overflow_rays, points_coarse, points_fine}.  ``near`` / ``far`` are cfg.min_depth /
    cfg.max_depth, ``surface_eps`` the fine band half-width (cfg.surface_eps).  Rays are processed ``chunk_rays`` at a
    time; the images do not depend on the chunking.  ``impl="fp32"`` runs the CUDA-core forward.  ``stages``: an
    optional dict that collects, per stage name (count0, emit0, forward0, composite0, then the same with 1), a list of
    (start, stop) CUDA events, one pair per chunk, for timing."""
    W, H = int(width), int(height)
    if W <= 0 or H <= 0:                                      # no ray to hand to the kernels, which check the rest
        raise _lib.VmbError(f"render_view: width and height must be >= 1 (got {W} x {H})")
    v = _View(sources, t_wc, K, W, H, n_coarse, n_fine, surface_eps, near, far)
    dev, a, S = v.dev, v.a, len(v.sources)
    f32, i32 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int32, device=dev)
    img = {"depth": torch.zeros(W, H, **f32), "colour": torch.zeros(W, H, 3, **f32),
           "opacity": torch.zeros(W, H, **f32), "instance": torch.full((W, H), -1, **i32)}
    a.depth, a.colour, a.opacity, a.instance = (_ptr(img[k]) for k in ("depth", "colour", "opacity", "instance"))
    stats = {"overflow_rays": 0, "points_coarse": 0, "points_fine": 0}
    n_pix, chunk = W * H, max(1, min(int(chunk_rays), W * H))
    hit_src = torch.empty(chunk, MAX_HITS, **i32)
    hit_t = torch.empty(chunk, MAX_HITS, 2, dtype=torch.float64, device=dev)
    hit_count = torch.empty(chunk, **i32)
    small = torch.zeros(1 + S, **i32)                         # overflow | src_total
    zstar = torch.empty(chunk, **f32)
    surf = torch.full((W, H), -1, **i32)                      # the coarse composite's surface sample, per pixel
    a.hit_src, a.hit_t, a.hit_count = _ptr(hit_src), _ptr(hit_t), _ptr(hit_count)
    a.overflow, a.src_total = _ptr(small), C.c_void_p(small.data_ptr() + 4)
    a.zstar = _ptr(zstar)

    def stage(name, fn):
        if stages is None:
            return fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        stages.setdefault(name, []).append((e0, e1))
        return r

    for r0 in range(0, n_pix, chunk):
        a.ray0, a.n_rays = r0, min(chunk, n_pix - r0)
        a.surf = C.c_void_p(surf.data_ptr() + 4 * r0)
        bufs = {}
        for p in (0, 1) if a.n_fine > 0 else (0,):
            setattr(a, "pass", p)
            stage(f"count{p}", lambda: v.call("vmb_render_count", "vmb_render_count"))
            host = small.cpu()                                # the one host sync of the pass: sizes the buffers
            if p == 0:
                stats["overflow_rays"] += int(host[0])
            totals = [int(x) for x in host[1:]]
            n = sum(totals)
            stats["points_coarse" if p == 0 else "points_fine"] += n
            pts, z = torch.empty(max(n, 1), 3, **f32), torch.empty(max(n, 1), **f32)
            base = torch.empty(a.n_rays, MAX_HITS, **i32)
            alpha, colour = torch.empty(max(n, 1), **f32), torch.empty(max(n, 1), 3, **f32)
            bufs[p] = (pts, z, base, alpha, colour)
            a.points, a.z, a.base = _ptr(pts), _ptr(z), _ptr(base)
            stage(f"emit{p}", lambda: v.call("vmb_render_emit", "vmb_render_emit"))
            stage(f"forward{p}", lambda: _forward(v.sources, totals, pts, alpha, colour, impl))
            a.z_coarse, a.alpha_coarse, a.colour_coarse, a.base_coarse = (
                _ptr(bufs[0][1]), _ptr(bufs[0][3]), _ptr(bufs[0][4]), _ptr(bufs[0][2]))
            if p == 1:
                a.z_fine, a.alpha_fine, a.colour_fine, a.base_fine = _ptr(z), _ptr(alpha), _ptr(colour), _ptr(base)
            stage(f"composite{p}", lambda: v.call("vmb_render_composite", "vmb_render_composite"))
        del bufs
    img["coarse_surface"] = surf
    if stats["overflow_rays"]:
        warnings.warn(f"render_view: {stats['overflow_rays']} rays hit more than {MAX_HITS} boxes; "
                      f"only the nearest {MAX_HITS} were rendered")
    return img, stats
