"""Bundle adjustment of keyframe poses against the object map on the GPU (K11).

Tracking fixes a frame's pose once; every later mapping frame samples that keyframe from it.  ``BundleAdjuster`` runs
pose-only passes against the frozen map: per pass

    K3 once per group on the objects' keyframe tables, in the camera frame, recording each draw's keyframe
      -> n_iter x [ vmb_ba_step per group on the iteration's ray slice -> vmb_ba_update (one Adam + Exp per frame) ]
      -> the refined poses written to the fp64 pose table, the frame store's slots and the background's copies

all on the device, so a pass can be captured as one CUDA graph (``capture`` / ``run``).  The rule is in
``csrc/k_ba.cuh``; ``oracle/ba_oracle.py`` restates it.  ``impl="layerwise"`` runs the step of every hidden-64/128/256
group on the tensor-core path (``vmb_ba_step_lw``, ``csrc/k_track_lw.cuh``), as ``Tracker`` does; ``impl="fused"``
also runs every hidden-32 group on the fused tile (``vmb_ba_step_fused``, ``csrc/k_track_fused.cuh``).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .ensemble import VmapEnsemble, _ptr, _stream
from .sampler import BatchedSampler, SamplerTables
from .track import _path, _rays_dir, _Slices, _step
from .utils import capture_graph


def fill_kf_frame(objs, store, kf_frame: np.ndarray, bg: bool = False) -> None:
    """``kf_frame`` [B, KF] on the host: the frame id of each keyframe index of each object (-1: none), from the
    shared-store objects' held slots or, for the ``do_bg`` background (``bg``), its own keyframe copies."""
    kf_frame[:] = -1
    for b, o in enumerate(objs):
        if bg:
            for f, j in o.kf_id_dict.items():
                kf_frame[b, j] = int(f)
        else:
            for j in range(kf_frame.shape[1]):
                if o._held[j]:
                    kf_frame[b, j] = int(store.frame_id[o.kf_store_slot[j]])


class PoseTables:
    """The int32 tables of a window of keyframe poses, in one pinned host buffer and its device twin: ``kf_frame(k)``
    [B_k, KF_k] of every group ``shapes[k] = (B_k, KF_k)``, the ``window`` (the distinct frame ids those hold without
    ``hold``, padded with -1 to ``max_win``), ``frame_of`` (the frame id of every store slot) and, with ``bg_kf``, the
    frame id of each of the ``do_bg`` background's keyframe copies.  Shared by ``BundleAdjuster`` and the joint mode of
    ``FrameLoop``."""

    def __init__(self, device, shapes: Sequence[Tuple[int, int]], max_win: int, bg_kf: int = 0):
        self.device, self.shapes, self.max_win, self.bg_kf = device, list(shapes), max_win, bg_kf
        self.cap = None
        self.window: List[int] = []

    def layout(self, store) -> bool:
        """Size the buffers for the store's capacity; True when they were (re)allocated."""
        cap = store.capacity
        if self.cap == cap:
            return False
        sizes = [b * kf for b, kf in self.shapes] + [self.max_win, cap] + ([self.bg_kf] if self.bg_kf else [])
        n = sum(sizes)
        self._host = torch.zeros(n, dtype=torch.int32)
        if torch.cuda.is_available():
            self._host = self._host.pin_memory()
        self._dev = torch.zeros(n, dtype=torch.int32, device=self.device)
        self._views, o = [], 0
        for s in sizes:
            self._views.append((o, s))
            o += s
        self.cap = cap
        self._uploaded = None
        return True

    def _h(self, k):
        o, s = self._views[k]
        return self._host[o:o + s]

    def _d(self, k):
        o, s = self._views[k]
        return self._dev[o:o + s]

    def kf_frame(self, k: int) -> torch.Tensor:
        return self._d(k)

    @property
    def window_dev(self) -> torch.Tensor:
        return self._d(len(self.shapes))

    @property
    def frame_of(self) -> torch.Tensor:
        return self._d(len(self.shapes) + 1)

    @property
    def bg_frame_of(self) -> torch.Tensor:
        return self._d(len(self.shapes) + 2)

    def prepare(self, store, fills, hold: int = 0, bg_group: Optional[int] = None) -> List[int]:
        """Fill every table on the host: ``fills[k](kf_frame)`` writes group k's [B_k, KF_k] table; the window and
        ``frame_of`` follow from them and the store; ``bg_group``: the group whose first row the background's table
        copies.  Returns the window (possibly empty).  Call ``layout`` first."""
        if self._uploaded is not None:
            self._uploaded.synchronize()       # the pinned buffer may still be the source of the last upload
        frames = set()
        for k, (b, kf) in enumerate(self.shapes):
            t = self._h(k).numpy().reshape(b, kf)
            fills[k](t)
            frames.update(int(f) for f in t.reshape(-1) if f >= 0)
        win = sorted(f for f in frames if f != hold)
        if len(win) > self.max_win:
            raise _lib.VmbError(f"pose window: {len(win)} frames exceed the window of {self.max_win}")
        ng = len(self.shapes)
        w = self._h(ng).numpy()
        w[:] = -1
        w[:len(win)] = win
        fo = self._h(ng + 1).numpy()
        fo[:] = -1
        for s, f in store.frame_id.items():
            if f is not None:
                fo[s] = int(f)
        if bg_group is not None:
            b, kf = self.shapes[bg_group]
            self._h(ng + 2).numpy()[:] = self._h(bg_group).numpy().reshape(b, kf)[0]
        self.window = win
        return win

    def upload(self) -> None:
        self._dev.copy_(self._host, non_blocking=True)
        if not torch.cuda.is_current_stream_capturing():
            if self._uploaded is None:
                self._uploaded = torch.cuda.Event()
            self._uploaded.record(torch.cuda.current_stream(self.device))


class _BaGroup(_Slices):
    """One ensemble's share of a pass: the shared-store objects of the mapping stack, or the ``do_bg`` background with
    its own keyframe copies.  Rows are those ``obj_ids`` names; ``kf_frame`` is the device table of their keyframes'
    frame ids, which ``BundleAdjuster`` provides."""

    def __init__(self, ens: VmapEnsemble, obj_ids: Sequence[Optional[int]], cfg, n_iter: int, bg: bool,
                 impl: str = "fp32"):
        ids = [None if i is None or int(i) < 0 else int(i) for i in obj_ids]
        assert len(ids) == ens.n_obj, "obj_ids must name every row of the ensemble (None / -1 = not an object)"
        self.ens, self.ids, self.bg, self.path = ens, ids, bg, _path(ens, impl)
        self.lw = self.path == "layerwise"      # the group runs on the layer-wise path
        self.rows = [r for r, i in enumerate(ids) if i is not None]
        B = len(self.rows)
        assert B > 0
        n1 = cfg.n_bins_cam2surface_bg if bg else cfg.n_bins_cam2surface
        self.smp = BatchedSampler(ens.device, n1, cfg.n_bins, cfg.surface_eps, cfg.stop_eps, cfg.min_depth)
        self.win = cfg.win_size_bg if bg else cfg.win_size                     # draws per iteration (train.py:196-199)
        self.n_pix_draw = cfg.n_samples_per_frame_bg if bg else cfg.n_samples_per_frame
        self.n_pix, self.S, self.KF = self.win * self.n_pix_draw, n1 + cfg.n_bins, cfg.keyframe_buffer_size
        self.n_draws = n_iter * self.win
        self._tiles("bundle adjustment")
        dev = ens.device
        self.rows_dev = torch.tensor(self.rows, dtype=torch.int32, device=dev)
        self.tables = SamplerTables(dev, B, kf_stride=0 if bg else self.KF)
        self.out = self.smp._outputs(B, self.n_draws * self.n_pix_draw, self.S, False)
        self.kf_out = torch.zeros(B, self.n_draws, dtype=torch.int32, device=dev)
        self._alloc_rows(B)

    def _alloc_rows(self, B: int) -> None:
        """The step's per-ray rows."""
        self.ray_rows = torch.zeros(B * self.n_pix, _lib.TRACK_PART, dtype=torch.float64, device=self.ens.device)

    def fill(self, objects: Dict[int, object], store, kf_frame: np.ndarray) -> None:
        """The sampler tables and ``kf_frame`` [B, KF] (frame id of each keyframe index, -1: none) on the host."""
        objs = [objects[self.ids[r]] for r in self.rows]
        if self.bg:
            self.tables.fill_objects([o.keyframe_set() for o in objs])
        else:
            from .vmap import keyframe_tables
            self.tables.fill_store(keyframe_tables(objs))
        fill_kf_frame(objs, store, kf_frame, self.bg)

    def sample(self, store, rays_dir, seed: int, counter) -> None:
        kw = dict(out=self.out, offset_dev=counter, camera_frame=True, kf_out=self.kf_out)
        if self.bg:
            self.smp.sample(None, self.n_draws, self.n_pix_draw, rays_dir, seed=seed, tables=self.tables, **kw)
        else:
            self.smp.sample_store(store, self.tables, self.n_draws, self.n_pix_draw, rays_dir, seed=seed, **kw)

    def bind(self, g, it: int) -> None:
        """vmb_ba_group for iteration ``it`` (0-based): rays [it * n_pix, (it + 1) * n_pix), draws
        [it * win, (it + 1) * win)."""
        super().bind(g, it)
        g.n_pix_draw = self.n_pix_draw
        g.kf_draw, g.kf_draw_stride = C.c_void_p(self.kf_out.data_ptr() + it * self.win * 4), self.n_draws
        g.kf_frame, g.kf_stride = _ptr(self.kf_frame), self.KF
        g.ray_rows, g.max_ray_rows = _ptr(self.ray_rows), self.ray_rows.shape[0]


class BundleAdjuster:
    """Pose-only passes over every keyframe the objects' keyframe tables hold, against the map's networks.

    ``groups``: ``[(VmapEnsemble, obj_ids), ...]`` with ``obj_ids[row]`` the instance id of each row (``None`` or -1
    for rows that are not objects), as ``track.groups_from_objects`` builds them; a group whose objects keep their own
    keyframe copies (the ``do_bg`` background) samples those.  ``n_iter`` iterations per pass in the mapping layout;
    rates default to ``cfg.pose_lr``; ``hold`` (the anchor frame) never moves.  ``record``: keep each pass's pose and
    gradient history per window entry (``pose_hist`` [n_iter+1, max_win, 4, 4], ``grad_hist`` [n_iter, max_win, 6]).
    ``impl``: ``"fp32"`` (K11 for every group), ``"layerwise"`` (the tensor-core path for hidden 64/128/256) or
    ``"fused"`` (as ``"layerwise"``, and the fused tile for hidden 32)."""

    def __init__(self, groups: Sequence[Tuple[VmapEnsemble, Sequence[Optional[int]]]], cfg, objects: Dict[int, object],
                 n_iter: int = 20, lr_rot: Optional[float] = None, lr_trans: Optional[float] = None, seed: int = 0,
                 hold: int = 0, record: bool = False, impl: str = "fp32"):
        if not 1 <= len(groups) <= _lib.TRACK_MAX_GROUPS:
            raise _lib.VmbError(f"BundleAdjuster: 1 .. {_lib.TRACK_MAX_GROUPS} groups")
        self.groups = []
        for e, ids in groups:
            named = [int(i) for i in ids if i is not None and int(i) >= 0]
            self.groups.append(_BaGroup(e, ids, cfg, n_iter, bg=getattr(objects[named[0]], "store", None) is None,
                                        impl=impl))
        self.impl = impl
        dev = self.groups[0].ens.device
        assert all(g.ens.device == dev for g in self.groups)
        self.device, self.cfg, self.n_iter, self.seed, self.hold = dev, cfg, n_iter, seed, hold
        self.lr_rot = cfg.pose_lr if lr_rot is None else lr_rot
        self.lr_trans = cfg.pose_lr if lr_trans is None else lr_trans
        self.rays_dir = _rays_dir(cfg, dev)
        self.max_win = min(_lib.BA_MAX_WIN, sum(len(g.rows) * g.KF for g in self.groups))
        f64 = dict(dtype=torch.float64, device=dev)
        self.adam = torch.zeros(self.max_win, 12, **f64)
        n_seg = sum(len(g.rows) * g.win for g in self.groups)
        self.scratch = torch.zeros(8 * n_seg + 6 * self.max_win, **f64)
        self.losses = torch.zeros(n_iter, **f64)
        self.status = torch.zeros(4, dtype=torch.int32, device=dev)
        self.pose_hist = torch.zeros(n_iter + 1, self.max_win, 4, 4, **f64) if record else None
        self.grad_hist = torch.zeros(n_iter, self.max_win, 6, **f64) if record else None
        self.counter = torch.zeros(1, dtype=torch.int64, device=dev)       # sampler draw counter, +1 per pass
        self.window: List[int] = []
        bg = [g for g in self.groups if g.bg]
        self.pose_tables = PoseTables(dev, [(len(g.rows), g.KF) for g in self.groups], self.max_win,
                                      bg[0].KF if bg else 0)
        self.graph: Optional[torch.cuda.CUDAGraph] = None

    # ---- the per-pass tables (PoseTables) ----------------------------------------------------------------------------
    def _layout(self, store) -> None:
        if self.pose_tables.layout(store):
            self.graph = None                  # a captured pass points at the old buffers
            for k, g in enumerate(self.groups):
                g.kf_frame = self.pose_tables.kf_frame(k)

    def prepare(self, store, objects: Dict[int, object]) -> List[int]:
        """Fill every table of the next pass on the host from the objects' keyframe tables; returns the window (the
        distinct frame ids those tables hold, without ``hold``), which may be empty."""
        self._layout(store)
        bg = [k for k, g in enumerate(self.groups) if g.bg]
        fills = [lambda t, g=g: g.fill(objects, store, t) for g in self.groups]
        self.window = self.pose_tables.prepare(store, fills, self.hold, bg[0] if bg else None)
        return self.window

    def _upload(self) -> None:
        self.pose_tables.upload()
        for g in self.groups:
            g.tables.upload()

    # ---- the pass ----------------------------------------------------------------------------------------------------
    def _enqueue(self, store, poses: torch.Tensor, objects: Dict[int, object], upload: bool = True) -> None:
        if upload:
            self._upload()
        for gi, g in enumerate(self.groups):
            g.sample(store, self.rays_dir, self.seed + 0x9e3779b9 * gi, self.counter)
        self.counter += 1
        pt = self.pose_tables
        targets = [(pt.frame_of, store.t_wc, store.capacity)]
        bg = [g for g in self.groups if g.bg]
        if bg:
            targets.append((pt.bg_frame_of, objects[bg[0].ids[bg[0].rows[0]]].t_wc_batch, bg[0].KF))
        a = _iterate(self.groups, self.n_iter, poses, pt.window_dev, self.max_win,
                     self.hold, self.adam, self.scratch, self.lr_rot, self.lr_trans, self.losses, self.status,
                     self.pose_hist, self.grad_hist, targets)
        self._args = a

    def run(self, store, poses: torch.Tensor, objects: Dict[int, object]) -> torch.Tensor:
        """One pass, eagerly: tables from ``objects`` ({id: sceneObject}, the background under 0), poses from and to
        the fp64 table ``poses`` [F, 4, 4] (row = frame id).  Returns the window; no host sync."""
        win = self.prepare(store, objects)
        if win:
            self._enqueue(store, poses, objects)
        return win

    def capture(self, store, poses: torch.Tensor, objects: Dict[int, object]) -> None:
        """Capture the pass as one CUDA graph for this object set and store; the warm-up and the capture change no
        pose, no store pose and no draw counter."""
        self.prepare(store, objects)
        bg = [objects[g.ids[g.rows[0]]].t_wc_batch for g in self.groups if g.bg]
        self.graph = capture_graph(self.device, lambda upload: self._enqueue(store, poses, objects, upload=upload),
                                   [poses, store.t_wc, self.counter] + bg)
        self._graph_key = (store, store.t_wc.data_ptr(), poses.data_ptr())

    def replay(self, store, poses: torch.Tensor, objects: Dict[int, object]) -> List[int]:
        """Replay the captured pass with this pass's tables; same results as ``run``."""
        if self.graph is None:
            raise _lib.VmbError("BundleAdjuster.replay: no graph for this object set and store; capture() first")
        assert self._graph_key == (store, store.t_wc.data_ptr(), poses.data_ptr()), "captured on other buffers"
        win = self.prepare(store, objects)
        if self.graph is None:                 # the store grew in between
            raise _lib.VmbError("BundleAdjuster.replay: the store grew since the capture; capture() again")
        if win:
            self._upload()
            self.graph.replay()
        return win


def _iterate(groups, n_iter, poses, window, n_win, hold, adam, scratch, lr_rot, lr_trans, losses, status,
             pose_hist=None, grad_hist=None, targets=()):
    """n_iter x [vmb_ba_step per group -> vmb_ba_update] on the groups' sample buffers."""
    a = ba_args(groups, n_iter, poses, window, n_win, hold, adam, scratch, lr_rot, lr_trans, losses, status,
                pose_hist, grad_hist, targets)
    e0 = groups[0].ens
    for it in range(n_iter):
        a.iter = it + 1
        for gi, g in enumerate(groups):
            g.bind(a.group[gi], it)
        for gi, g in enumerate(groups):
            _step(g, a, gi, ba=True)
        ba_update(e0, a)
    return a


def ba_update(ens: VmapEnsemble, a) -> None:
    """vmb_ba_update: one Adam + Exp over the window from the rows the iteration's steps wrote."""
    with ens._on_device():
        _lib.check(ens._handle, ens.lib.vmb_ba_update(ens._handle, C.byref(a), _stream()), "vmb_ba_update")


def ba_args(groups, n_iter, poses, window, n_win, hold, adam, scratch, lr_rot, lr_trans, losses, status,
            pose_hist=None, grad_hist=None, targets=()):
    """The vmb_ba_args of a pass over ``groups`` (each group's slice is bound per iteration by ``g.bind``)."""
    a = _lib.BaArgs()
    a.n_groups, a.n_iter = len(groups), n_iter
    a.poses, a.n_poses = _ptr(poses), poses.shape[0]
    a.window, a.n_win, a.hold = _ptr(window), n_win, hold
    a.adam, a.scratch, a.scratch_len = _ptr(adam), _ptr(scratch), scratch.numel()
    a.lr_rot, a.lr_trans, a.beta1, a.beta2, a.eps = lr_rot, lr_trans, 0.9, 0.999, 1e-8
    e0 = groups[0].ens
    a.colour_scaling, a.opacity_scaling = e0.colour_scaling, e0.opacity_scaling
    a.loss, a.status = _ptr(losses), _ptr(status)
    a.pose_hist, a.grad_hist = _ptr(pose_hist), _ptr(grad_hist)
    for t, (frame_of, t_wc, n) in enumerate(targets):
        a.target[t].frame_of, a.target[t].t_wc, a.target[t].n = _ptr(frame_of), _ptr(t_wc), n
    return a


class BaSampleGroup(_BaGroup):
    """A group fed with given samples instead of the sampler (tests, timing): ``batch`` holds [B, n_iter * R] rays of
    camera-frame points (``pcs`` [B,N,S,3]) and targets for the rows ``rows`` of ``ens``; ``kf_draw`` [B, N / n_pix_draw]
    the keyframe index of each draw and ``kf_frame`` [B, KF] the frame id of each keyframe index (-1: none); ``impl``
    as ``BundleAdjuster``'s."""

    def __init__(self, ens: VmapEnsemble, rows: Sequence[int], batch: Dict[str, torch.Tensor], n_iter: int,
                 n_pix_draw: int, kf_draw, kf_frame, impl: str = "fp32"):
        self.ens, self.rows, self.path = ens, list(rows), _path(ens, impl)
        self.lw = self.path == "layerwise"      # the group runs on the layer-wise path
        B, N, S = batch["pcs"].shape[:3]
        assert B == len(self.rows) and N % n_iter == 0 and (N // n_iter) % n_pix_draw == 0
        self.n_pix, self.S, self.n_pix_draw = N // n_iter, S, n_pix_draw
        self.win, self.n_draws = self.n_pix // n_pix_draw, N // n_pix_draw
        self._upload(self.rows, batch)
        dev = ens.device
        self.kf_out = torch.as_tensor(kf_draw, dtype=torch.int32).to(dev).contiguous()
        self.kf_frame = torch.as_tensor(kf_frame, dtype=torch.int32).to(dev).contiguous()
        self.KF = self.kf_frame.shape[1]
        assert self.kf_out.shape == (B, self.n_draws) and self.kf_frame.shape[0] == B
        self._tiles("bundle adjustment")
        self._alloc_rows(B)


def ba_samples(groups: Sequence[BaSampleGroup], poses, window: Sequence[int], n_iter: int, lr_rot: float,
               lr_trans: float, hold: int = 0, record: bool = True):
    """The pass on given samples: returns dict(poses [F,4,4] (the table after the pass), losses [n_iter], status, and
    with ``record`` pose_hist [n_iter+1,n_win,4,4], grad_hist [n_iter,n_win,6]) as device tensors.  ``window`` is
    used as given (padding -1 allowed)."""
    dev = groups[0].ens.device
    f64 = dict(dtype=torch.float64, device=dev)
    P = torch.as_tensor(np.asarray(poses.cpu() if torch.is_tensor(poses) else poses, np.float64)).to(dev).contiguous()
    n_win = len(window)
    n_seg = sum(len(g.rows) * g.win for g in groups)
    out = {"poses": P, "losses": torch.zeros(n_iter, **f64), "status": torch.zeros(4, dtype=torch.int32, device=dev)}
    if record:
        out["pose_hist"] = torch.zeros(n_iter + 1, n_win, 4, 4, **f64)
        out["grad_hist"] = torch.zeros(n_iter, n_win, 6, **f64)
    win = torch.tensor(list(window), dtype=torch.int32, device=dev)
    _iterate(list(groups), n_iter, P, win, n_win, hold, torch.zeros(n_win, 12, **f64),
             torch.zeros(8 * n_seg + 6 * n_win, **f64), lr_rot, lr_trans, out["losses"], out["status"],
             out.get("pose_hist"), out.get("grad_hist"))
    return out
