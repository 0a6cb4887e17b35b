"""Online SLAM on the GPU: track each new frame against the map of the frames before it, then map it from that pose.

``Slam`` composes the package's public pieces, one RGB-D + instance frame at a time:

    predict (fp64 device torch) -> FrameStore.ingest (K ingest) -> Tracker (K3 + K10) -> write the pose
      -> sceneObject keyframes (the reference's policy, vmap.py:208-268) and new objects (update_vmap)
      -> FrameLoop (K3 + the mapping steps, with the Background model when ``do_bg``)

Every pose stays a device tensor.  The host reads, per frame, the ingest's keep flags and boxes (one small copy the
keyframe tables need anyway) and, when objects are inserted, what ``update_vmap`` and a new ``FrameLoop`` read.  The
rules that are the package's own (INTEGRATION.md section 5):

* motion model: frame 0 takes the caller's anchor ``T_init``, frame 1 predicts T_0, and frame k >= 2 predicts the
  constant-velocity pose T_{k-1} (T_{k-2}^-1 T_{k-1}), all in fp64;
* a frame is *lost* when no mapped object is visible in it or when the tracker's status word reports a non-finite
  value; it keeps the predicted pose, is flagged, and the sequence goes on;
* an object is tracked from the frame after its insertion (it needs one mapping frame to have a network);
* with ``do_bg`` off the background (id 0) is an ordinary object of the stack, as in the reference, and it is not
  tracked: the tracker samples the background only as a model of its own.

Tracking replays a captured graph once the tracked set has stayed the same for a frame: a frame whose set changed is
tracked eagerly (``Tracker.track``), the next frame with that set captures (one more eager frame for the warm-up, a
device synchronise and the capture) and later frames replay.  ``track_modes`` records which of the three each frame was.

The frame store starts small and doubles when a new frame finds no free slot, up to ``max_n_models *
keyframe_buffer_size + 1`` slots: every object holds at most ``keyframe_buffer_size`` keyframe slots, and the live
frame holds one.  Growing reallocates the frames, so both captured graphs are captured again.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from . import _lib
from .frame import Background, FrameLoop
from .keyframes import FrameStore
from .sampler import BatchedSampler
from .track import Tracker, _rays_dir, groups_from_objects
from .vmap import keyframe_tables, sceneObject

# the tracker's sampler key: tracking frame k must not reuse the Philox streams that mapped frame k - 1
_TRACK_SEED = 0x2545F491


def _inv_se3(T: torch.Tensor) -> torch.Tensor:
    R, t = T[:3, :3], T[:3, 3]
    out = torch.eye(4, dtype=T.dtype, device=T.device)
    out[:3, :3] = R.T
    out[:3, 3] = -(R.T @ t)
    return out


def tracker_groups(groups, do_bg: bool):
    """``groups`` (``[(VmapEnsemble, obj_ids)]``) as the Tracker takes them.  The background (id 0) is tracked only as
    the separate background model of a ``do_bg`` map; with ``do_bg`` off it is an ordinary object network and its row
    is left out."""
    return [(e, [None if i is None or int(i) < 0 or (int(i) == 0 and not do_bg) else int(i) for i in ids])
            for e, ids in groups]


class Slam:
    """Online mapping and tracking of one sequence on one GPU.

    ``track=False`` maps from the poses the caller passes (the reference's train.py loop on the package's GPU path);
    ``map=False`` only localises, against ``groups`` (``[(VmapEnsemble, obj_ids)]`` as ``Tracker`` takes them, e.g. a
    map loaded from checkpoints).  ``graph``: replay the tracking frame and the mapping frame as CUDA graphs while the
    tracked set and the object set stay the same.  ``n_track_iter`` / ``lr_rot`` / ``lr_trans``: the tracker's
    iterations and rates (default ``cfg.pose_lr``).  ``store_capacity``: the frame store's initial number of slots (it
    grows on demand).  ``timing``: record CUDA events at the phase boundaries of every frame (``phase_times``)."""

    def __init__(self, cfg, T_init=None, track: bool = True, map: bool = True, groups=None, graph: bool = True,
                 n_track_iter: int = 20, lr_rot: Optional[float] = None, lr_trans: Optional[float] = None,
                 seed: int = 0, max_frames: int = 100000, background_cls: Sequence[int] = (), bbox_scale: float = 0.2,
                 store_capacity: Optional[int] = None, max_id: int = 4096, timing: bool = False):
        if not track and not map:
            raise ValueError("Slam: nothing to do with track=False and map=False")
        if not map and groups is None:
            raise ValueError("Slam(map=False) localises against a given map: pass groups")
        self.cfg, self.do_track, self.do_map, self.graph = cfg, track, map, graph
        self.device = torch.device(cfg.data_device)
        dev = self.device
        self.seed, self.n_track_iter = seed, n_track_iter
        self.track_kw = dict(n_iter=n_track_iter, lr_rot=lr_rot, lr_trans=lr_trans, seed=seed + _TRACK_SEED)
        self.background_cls, self.bbox_scale = list(background_cls), bbox_scale
        # localisation holds only the live frame; mapping holds each object's keyframes (see the module docstring)
        self.max_slots = cfg.max_n_models * cfg.keyframe_buffer_size + 1 if map else 1
        cap = min(store_capacity or 4 * cfg.keyframe_buffer_size + 1, self.max_slots)
        self.store = FrameStore(cfg.W, cfg.H, cap, device=dev, max_id=max_id)
        self.rays_dir = _rays_dir(cfg, dev)
        f64 = dict(dtype=torch.float64, device=dev)
        self.T_init = None if T_init is None else torch.as_tensor(T_init, dtype=torch.float64).to(dev).reshape(4, 4)
        # the per-frame record, on the device until ``result``
        self.poses = torch.zeros(max_frames, 4, 4, **f64)
        self.lost = torch.zeros(max_frames, dtype=torch.bool, device=dev)
        self.track_loss = torch.full((max_frames,), float("nan"), **f64)
        self.map_loss = torch.full((max_frames,), float("nan"), dtype=torch.float32, device=dev)
        self.tracked_ids: List[List[int]] = []
        self.track_modes: List[str] = []                 # per frame: "", "eager", "capture" or "replay"
        self.inserted: Dict[int, int] = {}               # object id -> frame it was inserted at
        self.k = 0
        self.timing, self.events = timing, []
        # the map
        self.objects: Dict[int, sceneObject] = {}         # objects of the packed stack (the reference's obj_dict)
        self.scene_bg: Optional[sceneObject] = None
        self.optimiser = None
        self.ens = self.loop = None
        self.tracker: Optional[Tracker] = None
        self._tracked_set = None
        if not map:
            groups = tracker_groups(groups, cfg.do_bg)
            self.tracker = Tracker(groups, cfg, **self.track_kw)
            self.mapped = {int(i) for _, ids in groups for i in ids if i is not None and int(i) >= 0}
        else:
            self.mapped = set()
            self.obj_sampler = BatchedSampler(dev, cfg.n_bins_cam2surface, cfg.n_bins, cfg.surface_eps, cfg.stop_eps,
                                              cfg.min_depth)
            self.bg_sampler = BatchedSampler(dev, cfg.n_bins_cam2surface_bg, cfg.n_bins, cfg.surface_eps,
                                             cfg.stop_eps, cfg.min_depth) if cfg.do_bg else None

    # ---- per frame -----------------------------------------------------------------------------------------------
    def _predict(self) -> torch.Tensor:
        k = self.k
        if k == 0:
            if self.T_init is None:
                raise ValueError("Slam: frame 0 needs the anchor pose T_init")
            return self.T_init.clone()
        if k == 1:
            return self.poses[0].clone()
        a, b = self.poses[k - 2], self.poses[k - 1]
        return b @ (_inv_se3(a) @ b)

    def step(self, rgb, depth, inst, cls=None, T_wc=None) -> int:
        """Process the next frame (images [W, H]: rgb uint8 [.., 3], depth metres, instance and class ids).  ``T_wc``:
        the frame's pose when ``track=False`` (ignored otherwise).  Returns the frame index."""
        k, cfg, dev = self.k, self.cfg, self.device
        if k >= self.poses.shape[0]:
            raise _lib.VmbError(f"Slam: more than max_frames={self.poses.shape[0]} frames")
        if not self.do_track:
            if T_wc is None:
                raise ValueError("Slam(track=False) maps from given poses: pass T_wc")
            T_pred = torch.as_tensor(T_wc, dtype=torch.float64).to(dev).reshape(4, 4)
        else:
            T_pred = self._predict()
        if self.store.n_used == self.store.capacity:
            self._grow()
        store = self.store
        self._mark(new_frame=True)
        slot, _, _ = store.ingest(rgb, depth, inst, T_pred, frame_id=k, cls=cls, background_cls=self.background_cls,
                                  bbox_scale=self.bbox_scale)
        # the one host read of the frame: keep flags and boxes of the kept instances (the keyframe tables' input)
        kb = torch.cat([store.stats[:, 7:8].float(), store.bbox], 1).cpu()
        visible = {int(i): kb[i, 1:] for i in torch.nonzero(kb[:, 0]).flatten().tolist()}
        self._mark()
        pose = T_pred
        ids = sorted(i for i in visible if i in self.mapped)
        self.tracked_ids.append(ids if self.do_track and (k > 0 or not self.do_map) else [])
        self.track_modes.append("")
        if self.do_track and (k > 0 or not self.do_map):
            if not ids:
                self.lost[k] = True
            else:
                pose = self._track(slot, T_pred, ids)
                bad = (self.tracker.status[0] & _lib.VMB_ST_NONFINITE) != 0
                self.lost[k] = bad
                pose = torch.where(bad, T_pred, pose)
                self.track_loss[k] = self.tracker.losses[-1]
            store.t_wc[slot] = pose.to(torch.float32)       # every consumer of the frame reads the store's pose
        self.poses[k] = pose
        self._mark()
        if self.do_map:
            self._map_frame(slot, k, visible, pose)
        store.release(slot)
        self._mark()
        self.k += 1
        return k

    def _mark(self, new_frame: bool = False) -> None:
        if self.timing:
            if new_frame:
                self.events.append([])
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.events[-1].append(e)

    def phase_times(self) -> dict:
        """With ``timing``: per frame, device milliseconds of ``ingest`` (with the keep-flag read), ``track``,
        ``bookkeeping`` (keyframes, insertion, tables: host work the device waits for) and ``map``, and ``frame``."""
        torch.cuda.synchronize(self.device)
        out = {k: [] for k in ("ingest", "track", "bookkeeping", "map", "frame")}
        for ev in self.events:
            d = [a.elapsed_time(b) for a, b in zip(ev[:-1], ev[1:])]
            if len(d) == 3:                                # no mapping mark (map=False)
                d = d[:2] + [d[2], 0.0]
            for key, v in zip(("ingest", "track", "bookkeeping", "map"), d):
                out[key].append(v)
            out["frame"].append(ev[0].elapsed_time(ev[-1]))
        return out

    def _track(self, slot: int, T_pred: torch.Tensor, ids: List[int]) -> torch.Tensor:
        tr = self.tracker
        tr.status.zero_()                                 # the status word is sticky: judge this frame alone
        if not self.graph or ids != self._tracked_set:    # a new set: eager now, capture if it is still there next frame
            self._tracked_set = list(ids)
            self.track_modes[-1] = "eager"
            pose, _ = tr.track(self.store, slot, T_pred, ids=ids)
            return pose
        if tr.graph is None:
            tr.capture(self.store, slot, T_pred, ids=ids)
            self.track_modes[-1] = "capture"
        else:
            self.track_modes[-1] = "replay"
        pose, _ = tr.run(self.store, slot, T_pred)
        return pose

    def _grow(self) -> None:
        """No free slot for the new frame: double the store (up to ``max_slots``) and drop the graphs captured on it."""
        cap = self.store.capacity
        if cap >= self.max_slots:
            raise _lib.VmbError(f"Slam: the frame store holds its maximum of {self.max_slots} frames")
        self.store.grow(min(2 * cap, self.max_slots))
        if self.loop is not None:
            self.loop.graph = None                        # FrameLoop.run captures again
        if self.tracker is not None:
            self.tracker.graph, self.tracker._graph_keep = None, None

    # ---- mapping (train.py:104-326 on the package's GPU path) --------------------------------------------------------
    def _map_frame(self, slot: int, k: int, visible: Dict[int, torch.Tensor], pose: torch.Tensor) -> None:
        cfg, store = self.cfg, self.store
        pose32 = pose.to(torch.float32)
        new = False
        for obj_id, bbox in sorted(visible.items()):
            if obj_id == -1:
                continue
            if cfg.do_bg and obj_id == 0:
                if self.scene_bg is None:
                    self.scene_bg = sceneObject(cfg, 0, *self._bg_images(slot), bbox, pose32, k)
                    self.inserted[0] = k
                    new = True
                else:
                    self.scene_bg.append_keyframe(*self._bg_images(slot), bbox, pose32, k)
            elif obj_id in self.objects:
                self.objects[obj_id].append_keyframe(None, None, None, bbox, pose32, k, frame_slot=slot)
            elif len(self.objects) < cfg.max_n_models:
                self.objects[obj_id] = sceneObject(cfg, obj_id, None, None, None, bbox, pose32, k, store=store,
                                                   frame_slot=slot)
                self.inserted[obj_id] = k
                new = True
        if not self.objects:
            return
        if new:
            self._restack()
        self.loop.set_store_tables(keyframe_tables(list(self.objects.values())))
        if self.loop.bg is not None:
            self.loop.set_background(self.scene_bg.keyframe_set())
        self._mark()
        losses = self.loop.run() if self.graph else self.loop.run_eager()
        self.map_loss[k] = losses[-1]

    def _bg_images(self, slot: int):
        """The background's own keyframe copies (per-object buffers, as ``Background`` samples them): rgb, depth and
        the state image of train.py:121-128 (1 = background, 2 = unknown), read from the store slot on the device."""
        inst = self.store.inst[slot]
        state = torch.zeros_like(inst, dtype=torch.uint8)
        state[inst == 0] = 1
        state[inst == -1] = 2
        return self.store.rgbx[slot, :, :, :3], self.store.depth[slot], state

    def _restack(self) -> None:
        """New objects: re-stack with update_vmap (train.py:178-182; Adam restarts for every object, as there), and
        rebuild the FrameLoop and the Tracker groups.  Both replace their captured graphs."""
        from . import utils
        cfg, dev = self.cfg, self.device
        if self.optimiser is None:
            self.optimiser = torch.optim.AdamW([torch.zeros((), requires_grad=True)], lr=cfg.learning_rate,
                                               weight_decay=cfg.weight_decay)
        objs = list(self.objects.values())
        utils.update_vmap([o.trainer.fc_occ_map for o in objs], self.optimiser)
        utils.update_vmap([o.trainer.pe for o in objs], self.optimiser)
        self.ens = self.optimiser._vmb_stack.ens
        bg = None
        if self.scene_bg is not None:
            from .lazy import ensemble_for_modules
            bg_ens = ensemble_for_modules(self.scene_bg.trainer.fc_occ_map, self.scene_bg.trainer.pe)
            bg = Background(bg_ens, self.bg_sampler, n_frames=cfg.n_iter_per_frame * cfg.win_size_bg,
                            n_pix=cfg.n_samples_per_frame_bg)
        old = self.loop
        self.loop = FrameLoop(self.ens, self.obj_sampler, cfg.n_iter_per_frame * cfg.win_size,
                              cfg.n_samples_per_frame, cfg.n_iter_per_frame, self.rays_dir, store=self.store,
                              kf_stride=cfg.keyframe_buffer_size, seed=self.seed, background=bg)
        if old is not None:
            self.loop.counter.copy_(old.counter)          # the sampler's draw counter runs on across re-stacks
        if self.do_track:
            self._rebuild_tracker()

    def _rebuild_tracker(self) -> None:
        objs = list(self.objects.values()) + ([self.scene_bg] if self.scene_bg is not None else [])
        groups = tracker_groups(groups_from_objects(objs), self.cfg.do_bg)
        old = self.tracker
        self.tracker = Tracker(groups, self.cfg, **self.track_kw)
        if old is not None:
            self.tracker.counter.copy_(old.counter)        # the tracker's draw counter runs on too
        self._tracked_set = None
        self.mapped = {i for _, ids in groups for i in ids if i is not None}

    # ---- the record --------------------------------------------------------------------------------------------------
    def result(self) -> dict:
        """The per-frame record read back (one copy at the end): ``poses`` [N, 4, 4] fp64, ``lost`` [N] bool,
        ``track_loss`` [N] fp64 (the tracker's last iteration; nan where not tracked), ``map_loss`` [N] (the last
        mapping iteration; nan where not mapped), ``tracked_ids``, ``inserted`` {object id: frame}, ``track_modes``
        and the frame store's final ``store_capacity``."""
        n = self.k
        return {"poses": self.poses[:n].cpu().numpy(), "lost": self.lost[:n].cpu().numpy(),
                "track_loss": self.track_loss[:n].cpu().numpy(), "map_loss": self.map_loss[:n].cpu().numpy(),
                "tracked_ids": [list(i) for i in self.tracked_ids], "inserted": dict(self.inserted),
                "track_modes": list(self.track_modes), "store_capacity": self.store.capacity}
