"""Track the camera pose of a new RGB-D frame against the object map on the GPU (K10).

The reference never estimates a pose: it reads GT poses (dataset.py:135) or takes them from an external tracker in
live mode.  ``Tracker`` closes that loop with the networks the map already has.  Per frame:

    K3 once per group on the new frame in the camera frame (one keyframe: the frame's slot and each object's box
      from this frame's ingest; the full frame for the background)  -> camera-frame points q
      -> n_iter x [ vmb_track_step per group on the iteration's ray slice -> vmb_track_update (Adam + Exp) ]

all on the device, so the loop can be captured as one CUDA graph (``capture`` / ``run``) as ``FrameLoop`` does for a
mapping frame.  The rule (points, loss, per-object empty masks, gradient, update) is in ``csrc/k_track.cuh``;
``oracle/track_oracle.py`` restates it.

``impl="layerwise"`` runs the step of every hidden-64/128/256 group on the tensor-core path instead
(``vmb_track_step_lw``, ``csrc/k_track_lw.cuh``: the same rule, the network in fp16 on wgmma GEMMs); hidden-32 groups
stay on K10.  ``impl="fused"`` does the same for hidden 64/128/256 and runs every hidden-32 group on the fused wgmma
tile (``vmb_track_step_fused``, ``csrc/k_track_fused.cuh``: the same rule, one launch for all the group's objects).  In
iMAP mode (``cfg.imap_mode``) id 0 is the whole-scene model and is sampled as an object.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .ensemble import VmapEnsemble, _ptr, _stream
from .sampler import BatchedSampler, KeyframeTables, SamplerTables
from .utils import capture_graph

IMPLS = ("fp32", "layerwise", "fused")


def _path(ens: VmapEnsemble, impl: str) -> str:
    """Where ``impl`` runs this ensemble's step: ``"fp32"`` (K10 / K11), ``"layerwise"`` (hidden 64/128/256 on the
    layer-wise tensor-core path, with "layerwise" or "fused") or ``"fused"`` (hidden 32 on the fused tile, with
    "fused").  A hidden-32 ensemble without its fp16 image cannot take the fused path: that raises."""
    if impl not in IMPLS:
        raise ValueError(f"tracking impl must be one of {IMPLS}, not {impl!r}")
    if impl == "fp32":
        return "fp32"
    if ens.hidden == 32:
        if impl == "layerwise":
            return "fp32"
        if ens.image is None:
            raise _lib.VmbError("tracking impl 'fused': the hidden-32 ensemble has no fp16 weight image")
        return "fused"
    return "layerwise" if ens.image is not None else "fp32"


def _step(g, a, gi: int, ba: bool) -> None:
    """The step of group ``gi`` on K10 / K11 or on the group's tensor-core path."""
    e = g.ens
    with e._on_device():
        if g.path != "fp32":
            if g.path == "fused":
                fn = e.lib.vmb_ba_step_fused if ba else e.lib.vmb_track_step_fused
            else:
                fn = e.lib.vmb_ba_step_lw if ba else e.lib.vmb_track_step_lw
            _lib.check(e._handle, fn(e._handle, C.byref(a), gi, _ptr(e.image), _stream()), fn.__name__)
        else:
            fn = e.lib.vmb_ba_step if ba else e.lib.vmb_track_step
            _lib.check(e._handle, fn(e._handle, C.byref(a), gi, _stream()), fn.__name__)


def _rays_dir(cfg, device) -> torch.Tensor:
    """cameraInfo.rays_dir_cache [W,H,3] = ((u-cx)/fx, (v-cy)/fy, 1) (vmap.py:494-524)."""
    u = (torch.arange(cfg.W, device=device) - cfg.cx) / cfg.fx
    v = (torch.arange(cfg.H, device=device) - cfg.cy) / cfg.fy
    d = torch.ones((cfg.W, cfg.H, 3), device=device)
    d[:, :, 0] = u[:, None]
    d[:, :, 1] = v
    return d.contiguous()


class _Slices:
    """One ensemble's rows ``rows_dev`` and their sample buffers ``out``: [B, N] rays in slices of ``n_pix`` rays of
    ``S`` samples, one slice per iteration.  Shared by the tracking and the bundle-adjustment groups."""

    def _tiles(self, what: str) -> int:
        """Tiles per object of the step at this slice shape; raises when the hidden size cannot take S samples."""
        tiles = self.ens.lib.vmb_track_tiles(self.ens.hidden, self.n_pix, self.S)
        if tiles < 0:
            raise _lib.VmbError(f"{what}: hidden {self.ens.hidden} does not support {self.S} samples per ray")
        return tiles

    def _upload(self, rows: Sequence[int], batch: Dict[str, torch.Tensor]) -> None:
        """Given samples instead of the sampler's: ``batch`` for the ensemble rows ``rows`` to the device."""
        dev = self.ens.device
        self.out = {k: v.to(dev).contiguous() for k, v in batch.items()}
        self.out["mask_depth"] = self.out["mask_depth"].to(torch.uint8)
        self.rows_dev = torch.tensor(list(rows), dtype=torch.int32, device=dev)

    def bind(self, g, it: int) -> None:
        """The fields vmb_track_group and vmb_ba_group share, for iteration ``it`` (0-based): rays
        [it * n_pix, (it + 1) * n_pix) of every row."""
        e, o, R, S = self.ens, self.out, self.n_pix, self.S
        B, N = o["pcs"].shape[:2]
        g.hidden, g.n_obj, g.n_rows, g.rows = e.hidden, B, e.n_obj, _ptr(self.rows_dev)
        g.n_rays, g.n_samples = R, S
        g.pcs, g.pcs_stride = C.c_void_p(o["pcs"].data_ptr() + it * R * S * 12), N * S * 3
        g.z_vals, g.z_stride = C.c_void_p(o["z"].data_ptr() + it * R * S * 4), N * S
        g.gt_depth, g.gt_depth_stride = C.c_void_p(o["gt_depth"].data_ptr() + it * R * 4), N
        g.gt_colour, g.gt_colour_stride = C.c_void_p(o["gt_colour"].data_ptr() + it * R * 12), N * 3
        g.sem, g.sem_stride = C.c_void_p(o["sem"].data_ptr() + it * R), N
        g.mask_depth, g.mask_stride = C.c_void_p(o["mask_depth"].data_ptr() + it * R), N
        g.params, g.scale = _ptr(e.params), _ptr(e.scale)


class _Group(_Slices):
    """One ensemble's share of the tracking problem: its sampler, the rows tracked this frame and their buffers."""

    def __init__(self, ens: VmapEnsemble, obj_ids: Sequence[Optional[int]], cfg, n_pix: int, n_pix_bg: int,
                 n_iter: int, impl: str = "fp32"):
        ids = [None if i is None or int(i) < 0 else int(i) for i in obj_ids]
        assert len(ids) == ens.n_obj, "obj_ids must name every row of the ensemble (None / -1 = not an object)"
        self.ens, self.ids, self.path = ens, ids, _path(ens, impl)
        self.lw = self.path == "layerwise"      # the group runs on the layer-wise path
        self.bg = 0 in ids and not getattr(cfg, "imap_mode", 0)     # iMAP: id 0 is the scene model, an object
        assert not self.bg or [i for i in ids if i is not None] == [0], "the background (id 0) is a group of its own"
        n1 = cfg.n_bins_cam2surface_bg if self.bg else cfg.n_bins_cam2surface
        self.smp = BatchedSampler(ens.device, n1, cfg.n_bins, cfg.surface_eps, cfg.stop_eps, cfg.min_depth)
        self.n_pix = n_pix_bg if self.bg else n_pix
        self.S = n1 + cfg.n_bins
        self.n_iter = n_iter
        self.tiles = self._tiles("tracking")
        self.active: List[int] = []

    def set_active(self, rows: Sequence[int]) -> bool:
        """Track ``rows`` from now on; returns True when that changed the set (and so replaced every buffer)."""
        rows = list(rows)
        if rows == self.active:
            return False
        dev = self.ens.device
        self.active = rows
        B = len(rows)
        if B == 0:
            return True
        self.rows_dev = torch.tensor(rows, dtype=torch.int32, device=dev)
        self.ids_dev = torch.tensor([self.ids[r] for r in rows], dtype=torch.int64, device=dev)
        self.tables = SamplerTables(dev, B, kf_stride=1)
        self.out = self.smp._outputs(B, self.n_iter * self.n_pix, self.S, False)
        self._alloc_rows(B)
        return True

    def _alloc_rows(self, B: int) -> None:
        """The step's partial rows (``tiles`` per object) and the update's per-object loss terms."""
        dev = self.ens.device
        self.partials = torch.zeros(max(B * self.tiles, 1), _lib.TRACK_PART, dtype=torch.float64, device=dev)
        self.loss_terms = torch.zeros(B, 4, dtype=torch.float32, device=dev)

    def buffers(self):
        return (self.rows_dev, self.ids_dev, self.tables, self.out, self.partials, self.loss_terms)

    def fill_tables(self, slot: int) -> None:
        B = len(self.active)
        kt = KeyframeTables(np.full((B, 1), slot, np.int32), np.zeros((B, 1, 4), np.float32),
                            [self.ids[r] for r in self.active], np.ones(B, np.int32), np.zeros((B, 2), np.int32))
        self.tables.fill_store(kt)

    def boxes_to_device(self, store) -> None:
        """This frame's boxes straight from the ingest's device table into the sampler tables (no host read)."""
        B = len(self.active)
        dst = self.tables.dev.view(torch.int32)[B:B * 5].view(torch.float32).view(B, 4)
        if self.bg:                                     # built on the first (eager) frame, never inside a capture
            if getattr(self, "_full", None) is None or self._full_wh != (store.W, store.H):
                self._full = torch.tensor([0.0, float(store.W), 0.0, float(store.H)], device=dst.device)
                self._full_wh = (store.W, store.H)
            dst.copy_(self._full.expand(B, 4))
        else:
            dst.copy_(store.bbox.index_select(0, self.ids_dev))

    def bind(self, g, it: int) -> None:
        """vmb_track_group for iteration ``it`` (0-based): rays [it * n_pix, (it + 1) * n_pix)."""
        super().bind(g, it)
        g.partials, g.max_partials = _ptr(self.partials), self.partials.shape[0]
        g.loss_terms = _ptr(self.loss_terms)


class Tracker:
    """Pose tracking of a frame already ingested in a ``FrameStore`` against the map's networks.

    ``groups``: ``[(VmapEnsemble, obj_ids), ...]`` with ``obj_ids[row]`` the instance id of each row (``None`` or -1
    for rows that are not objects); the background (id 0) is a group of its own.  ``n_iter`` iterations of ``n_pix``
    rays per object (``n_pix_bg`` for the background); rates default to ``cfg.pose_lr``.  ``impl``: ``"fp32"`` (K10
    for every group), ``"layerwise"`` (the tensor-core path for hidden-64/128/256 groups, K10 for hidden 32) or
    ``"fused"`` (as ``"layerwise"``, and the fused tile for hidden-32 groups)."""

    def __init__(self, groups: Sequence[Tuple[VmapEnsemble, Sequence[Optional[int]]]], cfg, n_iter: int = 20,
                 n_pix: Optional[int] = None, n_pix_bg: Optional[int] = None, lr_rot: Optional[float] = None,
                 lr_trans: Optional[float] = None, seed: int = 0, record: bool = False, impl: str = "fp32"):
        if not 1 <= len(groups) <= _lib.TRACK_MAX_GROUPS:
            raise _lib.VmbError(f"Tracker: 1 .. {_lib.TRACK_MAX_GROUPS} groups")
        n_pix = cfg.n_per_optim if n_pix is None else n_pix
        n_pix_bg = cfg.n_per_optim_bg if n_pix_bg is None else n_pix_bg
        self.groups = [_Group(e, ids, cfg, n_pix, n_pix_bg, n_iter, impl) for e, ids in groups]
        self.impl = impl
        dev = self.groups[0].ens.device
        assert all(g.ens.device == dev for g in self.groups)
        self.device, self.cfg, self.n_iter, self.seed = dev, cfg, n_iter, seed
        self.lr_rot = cfg.pose_lr if lr_rot is None else lr_rot
        self.lr_trans = cfg.pose_lr if lr_trans is None else lr_trans
        f64 = dict(dtype=torch.float64, device=dev)
        self.rays_dir = _rays_dir(cfg, dev)
        self.pose = torch.eye(4, **f64)
        self.adam = torch.zeros(12, **f64)
        self.losses = torch.zeros(n_iter, **f64)
        self.status = torch.zeros(4, dtype=torch.int32, device=dev)
        self.pose_hist = torch.zeros(n_iter + 1, 4, 4, **f64) if record else None
        self.grad_hist = torch.zeros(n_iter, 6, **f64) if record else None
        self.counter = torch.zeros(1, dtype=torch.int64, device=dev)       # sampler draw counter, +1 per frame
        self.slot_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self._graph_keep = None

    # ---- which rows this frame tracks ------------------------------------------------------------------------------
    def select(self, ids: Sequence[int]) -> None:
        """Track the rows whose instance id is in ``ids``, plus the background if it is in a group."""
        want = set(int(i) for i in ids)
        changed = [g.set_active([r for r, i in enumerate(g.ids) if i is not None and (i in want or i == 0)])
                   for g in self.groups]
        if any(changed):                    # a captured graph points at the buffers of the set it was captured for
            self.graph, self._graph_keep = None, None
        if not any(g.active for g in self.groups):
            raise _lib.VmbError("Tracker: no map object is visible in this frame")

    def _live(self) -> List[_Group]:
        return [g for g in self.groups if g.active]

    def _set_pose(self, T_init) -> None:
        if torch.is_tensor(T_init) and T_init.is_cuda:
            self.pose.copy_(T_init.reshape(4, 4))
            return
        T = np.asarray(T_init.cpu() if torch.is_tensor(T_init) else T_init, np.float64).reshape(4, 4)
        if not np.all(np.isfinite(T)):
            raise _lib.VmbError("Tracker: the initial pose is not finite")
        self.pose.copy_(torch.from_numpy(T), non_blocking=False)

    def _call(self, fn, *args):
        e = self.groups[0].ens
        with e._on_device():
            _lib.check(e._handle, fn(*args), fn.__name__)

    # ---- the frame ---------------------------------------------------------------------------------------------------
    def _enqueue(self, store, upload: bool = True) -> None:
        live = self._live()
        for gi, g in enumerate(live):
            if upload:
                g.tables.upload()
            g.boxes_to_device(store)
            g.smp.sample_store(store, g.tables, self.n_iter, g.n_pix, self.rays_dir, seed=self.seed + 0x9e3779b9 * gi,
                               out=g.out, offset_dev=self.counter, camera_frame=True)
        self.counter += 1
        self._args = _iterate(live, self.n_iter, self.pose, self.adam, self.lr_rot, self.lr_trans, self.losses,
                              self.status, self.pose_hist, self.grad_hist)
        store.t_wc.index_copy_(0, self.slot_dev, self.pose.to(torch.float32)[None])

    def _prepare(self, store, slot: int, T_init) -> None:
        for g in self._live():
            g.fill_tables(slot)
        self.slot_dev.fill_(slot)
        self._set_pose(T_init)

    def track(self, store, slot: int, T_init, ids: Optional[Sequence[int]] = None):
        """Track frame ``slot`` of ``store`` (ingested) from ``T_init`` [4,4].  ``ids``: instance ids to track; by
        default those the last ingest kept (one small read of the keep flags).  On exit ``store.t_wc[slot]`` holds
        the tracked pose in fp32.  Returns (pose [4,4] fp64, losses [n_iter] fp64), device tensors, no host sync."""
        self.select(store.visible_objects().keys() if ids is None else ids)
        self._prepare(store, slot, T_init)
        self._enqueue(store)
        return self.pose.clone(), self.losses.clone()

    def capture(self, store, slot: int, T_init, ids: Optional[Sequence[int]] = None) -> None:
        """Capture the frame (sampling + every iteration) as one CUDA graph for the current set of tracked rows.  The
        warm-up and the capture do not advance the draw counter."""
        self.select(store.visible_objects().keys() if ids is None else ids)
        self._prepare(store, slot, T_init)
        self.graph = capture_graph(self.device, lambda upload: self._enqueue(store, upload=upload),
                                   [self.counter, store.t_wc[slot]])
        self._graph_store = store
        self._graph_keep = [g.buffers() for g in self._live()]     # alive as long as the graph that writes them

    def run(self, store, slot: int, T_init):
        """Replay the captured frame on frame ``slot`` for the rows tracked at capture; same results as ``track``.  A
        ``track`` or ``capture`` for another set of rows in between drops the graph: capture again."""
        if self.graph is None:
            raise _lib.VmbError("Tracker.run: no graph for the current set of tracked rows; capture() first")
        assert store is self._graph_store, "the graph was captured on another FrameStore"
        self._prepare(store, slot, T_init)
        for g in self._live():
            g.tables.upload()
        self.graph.replay()
        return self.pose.clone(), self.losses.clone()

    def loss_terms(self) -> Dict[int, torch.Tensor]:
        """Per tracked object: its last iteration's [L_depth, L_colour, L_opacity, total] (device tensors)."""
        return {g.ids[r]: g.loss_terms[k] for g in self._live() for k, r in enumerate(g.active)}


def _iterate(live, n_iter, pose, adam, lr_rot, lr_trans, losses, status, pose_hist=None, grad_hist=None):
    """n_iter x [vmb_track_step per group -> vmb_track_update] on the groups' sample buffers."""
    a = _lib.TrackArgs()
    a.n_groups, a.n_iter = len(live), n_iter
    a.pose, a.adam = _ptr(pose), _ptr(adam)
    a.lr_rot, a.lr_trans, a.beta1, a.beta2, a.eps = lr_rot, lr_trans, 0.9, 0.999, 1e-8
    a.colour_scaling, a.opacity_scaling = live[0].ens.colour_scaling, live[0].ens.opacity_scaling
    a.loss, a.status = _ptr(losses), _ptr(status)
    a.pose_hist, a.grad_hist = _ptr(pose_hist), _ptr(grad_hist)
    for it in range(n_iter):
        a.iter = it + 1
        for gi, g in enumerate(live):
            g.bind(a.group[gi], it)
        for gi, g in enumerate(live):
            _step(g, a, gi, ba=False)
        e = live[0].ens
        with e._on_device():
            _lib.check(e._handle, e.lib.vmb_track_update(e._handle, C.byref(a), _stream()), "vmb_track_update")
    return a


class SampleGroup(_Group):
    """A group fed with given samples instead of the sampler (tests, timing): ``batch`` holds [B, n_iter * n_pix]
    rays of camera-frame points (``pcs`` [B,N,S,3]) and targets for the rows ``rows`` of ``ens``; ``impl`` as
    ``Tracker``'s."""

    def __init__(self, ens: VmapEnsemble, rows: Sequence[int], batch: Dict[str, torch.Tensor], n_iter: int,
                 impl: str = "fp32"):
        self.ens, self.active, self.n_iter, self.path = ens, list(rows), n_iter, _path(ens, impl)
        self.lw = self.path == "layerwise"      # the group runs on the layer-wise path
        B, N, S = batch["pcs"].shape[:3]
        assert B == len(self.active) and N % n_iter == 0
        self.n_pix, self.S = N // n_iter, S
        self._upload(self.active, batch)
        self.tiles = self._tiles("tracking")
        self._alloc_rows(B)


def track_samples(groups: Sequence[SampleGroup], T_init, n_iter: int, lr_rot: float, lr_trans: float,
                  record: bool = True):
    """The tracking loop on given samples: returns dict(pose [4,4], losses [n_iter], and with ``record`` pose_hist
    [n_iter+1,4,4], grad_hist [n_iter,6]) as device fp64 tensors, plus the status word."""
    dev = groups[0].ens.device
    f64 = dict(dtype=torch.float64, device=dev)
    pose = torch.as_tensor(np.asarray(T_init.cpu() if torch.is_tensor(T_init) else T_init, np.float64)).to(dev)
    out = {"pose": pose.clone(), "losses": torch.zeros(n_iter, **f64),
           "status": torch.zeros(4, dtype=torch.int32, device=dev)}
    if record:
        out["pose_hist"] = torch.zeros(n_iter + 1, 4, 4, **f64)
        out["grad_hist"] = torch.zeros(n_iter, 6, **f64)
    _iterate(list(groups), n_iter, out["pose"], torch.zeros(12, **f64), lr_rot, lr_trans, out["losses"],
             out["status"], out.get("pose_hist"), out.get("grad_hist"))
    return out


def groups_from_objects(objects) -> List[Tuple[VmapEnsemble, List[Optional[int]]]]:
    """Tracker groups of drop-in ``sceneObject``s: one group per packed ensemble, each row named by the object bound
    to it (as ``render.sources_from_objects`` finds them)."""
    from .lazy import ensemble_for_modules
    by_ens: Dict[int, Tuple[VmapEnsemble, List[Optional[int]]]] = {}
    for obj in objects:
        t = obj.trainer
        ens = ensemble_for_modules(t.fc_occ_map, t.pe)
        row = t.fc_occ_map._vmb_binding[1]
        ent = by_ens.setdefault(id(ens), (ens, [None] * ens.n_obj))
        ent[1][row] = int(obj.obj_id)
    return list(by_ens.values())
