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
frame holds one.  Growing reallocates the frames, so the captured graphs are captured again.

With ``ba_every`` > 0, every ``ba_every`` frames a bundle-adjustment pass (``ba.BundleAdjuster``, K11) runs after the
mapping frame: ``n_ba_iter`` pose-only iterations against the frozen map move every keyframe pose the objects' keyframe
tables hold (never frame 0, the anchor), and the refined poses go to ``poses``, the store and the background's
copies, where the next mapping frames, the motion model, ``get_bound`` and meshing read them.  Its graph follows the
same eager / capture / replay pattern (``ba_modes``).

In iMAP mode (``cfg.imap_mode``) every pixel of a frame is instance 0 (dataset.py:95-96) and id 0 is the one
whole-scene network, an object of the stack as mapping builds it (``hidden_feature_size``, ``obj_scale``,
``n_bins_cam2surface``, ``n_per_optim``); it is tracked like any other object from the frame after its insertion, with
its box from the ingest.  ``track_impl`` / ``ba_impl`` choose the step of the tracker and the bundle adjuster:
``"layerwise"`` (the tensor-core path for hidden 64/128/256, the default in iMAP mode), ``"fp32"`` (K10 / K11, the
default otherwise) or ``"fused"`` (as ``"layerwise"``, and the vMAP objects' hidden-32 models on the fused wgmma tile;
in iMAP mode, which has no hidden-32 model, the same as ``"layerwise"``).

With ``joint_poses`` (iMAP mode only) every mapping iteration also moves the keyframe poses, as iMAP optimises its
network and keyframe poses together: the mapping frame runs ``FrameLoop``'s joint mode (``vmb_joint_step_lw``: the pose
rows come from the mapping step's own backward, no second forward), one Adam + Exp over the window of every keyframe the
model holds per iteration (never frame 0, the anchor), and the refined poses go to ``poses`` and the store, where the
motion model, ``get_bound``, meshing and bundle adjustment read them.  The pose Adam moments restart with every mapping
frame, as a bundle-adjustment pass's do.  ``joint_impl`` chooses the joint step: ``"layerwise"`` (the default, iMAP
mode) or ``"fused"`` (vMAP mode: ``vmb_joint_step_fused``, the objects' fused hidden-32 step with AdamW inside it, whose
PE backward also gives the pose rows; with ``do_bg`` the background model's joint step is the update's second group and
its keyframe copies receive the refined poses too).  In vMAP mode joint poses need ``joint_impl="fused"``.

On ScanNet sequences (``assoc``: one ``scannet.InstanceTracker`` for the whole sequence, vMAP mode with ``map=True``)
a frame's instance image comes from the instance association (utils.box_filter), which needs the frame's pose.  The
ids of the objects already mapped are known before the pose is, so per frame:

1. the prediction, and ``FrameStore.ingest`` of the **raw** ids (instance + 1) with the ScanNet background classes:
   the provisional labels;
2. tracking of the kept and mapped ids against the map, as above (each tracked object's full raw mask: no erosion and
   no -1 "unsure" pixels);
3. the association at the frame's final pose (the tracked one, the kept prediction of a lost frame, or the given pose
   with ``track=False``): the only call that changes the association state;
4. ``FrameStore.relabel`` of the slot from its labels and 2-D boxes (dataset.py:263-283), then keyframes, insertion,
   the background state image and mapping as above.

The association's clouds keep the poses they were merged at: bundle adjustment and joint poses do not re-pose them.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .frame import Background, FrameLoop, JointPoses
from .keyframes import FrameStore
from .ba import BundleAdjuster
from .sampler import BatchedSampler
from .track import Tracker, _rays_dir, groups_from_objects
from .vmap import keyframe_tables, sceneObject

# the tracker's sampler key: tracking frame k must not reuse the Philox streams that mapped frame k - 1
_TRACK_SEED = 0x2545F491
# the bundle adjuster's sampler key, distinct from the mapping frames' and the tracker's
_BA_SEED = 0x61C88647


def _inv_se3(T: torch.Tensor) -> torch.Tensor:
    R, t = T[:3, :3], T[:3, 3]
    out = torch.eye(4, dtype=T.dtype, device=T.device)
    out[:3, :3] = R.T
    out[:3, 3] = -(R.T @ t)
    return out


def tracker_groups(groups, do_bg: bool, imap: bool = False):
    """``groups`` (``[(VmapEnsemble, obj_ids)]``) as the Tracker takes them.  The background (id 0) is tracked only as
    the separate background model of a ``do_bg`` map; with ``do_bg`` off it is an ordinary object network and its row
    is left out.  In iMAP mode (``imap``) id 0 is the whole-scene model, the only object, and it is kept."""
    return [(e, [None if i is None or int(i) < 0 or (int(i) == 0 and not do_bg and not imap) else int(i) for i in ids])
            for e, ids in groups]


class Slam:
    """Online mapping and tracking of one sequence on one GPU.

    ``track=False`` maps from the poses the caller passes (the reference's train.py loop on the package's GPU path);
    ``map=False`` only localises, against ``groups`` (``[(VmapEnsemble, obj_ids)]`` as ``Tracker`` takes them, e.g. a
    map loaded from checkpoints).  ``graph``: replay the tracking frame and the mapping frame as CUDA graphs while the
    tracked set and the object set stay the same.  ``n_track_iter`` / ``lr_rot`` / ``lr_trans``: the tracker's
    iterations and rates (default ``cfg.pose_lr``).  ``store_capacity``: the frame store's initial number of slots (it
    grows on demand).  ``timing``: record CUDA events at the phase boundaries of every frame (``phase_times``).
    ``ba_every``: run a bundle-adjustment pass after the mapping frame of every ``ba_every``-th frame (0: never);
    ``n_ba_iter`` / ``ba_lr_rot`` / ``ba_lr_trans``: its iterations and rates (default ``cfg.pose_lr``).
    ``track_impl`` / ``ba_impl``: ``"fp32"``, ``"layerwise"`` or ``"fused"`` (see the module docstring; None:
    ``"layerwise"`` in iMAP mode, ``"fp32"`` otherwise).  ``joint_poses``: optimise the keyframe poses with the map in every mapping iteration
    (see the module docstring); ``joint_lr_rot`` / ``joint_lr_trans``: its rates (default ``cfg.pose_lr``);
    ``joint_impl``: ``None`` / ``"layerwise"`` (iMAP mode) or ``"fused"`` (vMAP mode).  ``assoc``: a
    ``scannet.InstanceTracker``, the one association state of a ScanNet sequence (see the module docstring); ``step``
    then takes raw ScanNet ids and classes, and ``background_cls`` defaults to ``scannet.BG_CLASSES``."""

    def __init__(self, cfg, T_init=None, track: bool = True, map: bool = True, groups=None, graph: bool = True,
                 n_track_iter: int = 20, lr_rot: Optional[float] = None, lr_trans: Optional[float] = None,
                 seed: int = 0, max_frames: int = 100000, background_cls: Sequence[int] = (), bbox_scale: float = 0.2,
                 store_capacity: Optional[int] = None, max_id: int = 4096, timing: bool = False, ba_every: int = 0,
                 n_ba_iter: int = 20, ba_lr_rot: Optional[float] = None, ba_lr_trans: Optional[float] = None,
                 track_impl: Optional[str] = None, ba_impl: Optional[str] = None, joint_poses: bool = False,
                 joint_lr_rot: Optional[float] = None, joint_lr_trans: Optional[float] = None,
                 joint_impl: Optional[str] = None, assoc=None):
        if assoc is not None and cfg.imap_mode:
            raise ValueError("Slam: assoc is the ScanNet instance association; in iMAP mode every pixel is instance 0 "
                             "and there is nothing to associate")
        if assoc is not None and not map:
            raise ValueError("Slam: assoc relabels the frames of a map being built: map=True (localisation on "
                             "ScanNet, map=False, is not supported)")
        if joint_impl not in (None, "layerwise", "fused"):
            raise ValueError(f"Slam: joint_impl must be None, 'layerwise' or 'fused', not {joint_impl!r}")
        if joint_impl == "fused" and cfg.imap_mode:
            raise ValueError("Slam: joint_impl='fused' is the vMAP objects' hidden-32 step; iMAP mode takes 'layerwise'")
        if joint_poses and not cfg.imap_mode and joint_impl != "fused":
            raise ValueError("Slam: joint_poses in vMAP mode needs joint_impl=\"fused\": the layer-wise joint step "
                             "runs the iMAP model, the vMAP objects' hidden-32 step is the fused one")
        if joint_poses and not map:
            raise ValueError("Slam: joint_poses refines the keyframe poses of a map being built: map=True")
        if not track and not map:
            raise ValueError("Slam: nothing to do with track=False and map=False")
        if ba_every < 0 or n_ba_iter < 1:
            raise ValueError("Slam: need ba_every >= 0 and n_ba_iter >= 1")
        if ba_every and not map:
            raise ValueError("Slam: bundle adjustment (ba_every > 0) refines the poses of a map being built: map=True")
        if not map and groups is None:
            raise ValueError("Slam(map=False) localises against a given map: pass groups")
        self.cfg, self.do_track, self.do_map, self.graph = cfg, track, map, graph
        self.device = torch.device(cfg.data_device)
        dev = self.device
        self.seed, self.n_track_iter = seed, n_track_iter
        self.imap = bool(cfg.imap_mode)
        default_impl = "layerwise" if self.imap else "fp32"
        self.track_kw = dict(n_iter=n_track_iter, lr_rot=lr_rot, lr_trans=lr_trans, seed=seed + _TRACK_SEED,
                             impl=track_impl or default_impl)
        self.assoc = assoc
        if assoc is not None and not len(background_cls):
            from .scannet import BG_CLASSES
            background_cls = [c for c in BG_CLASSES if c >= 0]
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
        # bundle adjustment (off: nothing is allocated or launched)
        self.ba_every = ba_every
        self.joint = JointPoses(self.poses, cfg.pose_lr if joint_lr_rot is None else joint_lr_rot,
                                cfg.pose_lr if joint_lr_trans is None else joint_lr_trans) if joint_poses else None
        self.ba_kw = dict(n_iter=n_ba_iter, lr_rot=ba_lr_rot, lr_trans=ba_lr_trans, seed=seed + _BA_SEED,
                          impl=ba_impl or default_impl)
        self.ba: Optional[BundleAdjuster] = None
        self.ba_loss = torch.full((max_frames,), float("nan"), **f64) if ba_every else None
        self.ba_frames: List[List[int]] = []
        self.ba_modes: List[str] = []                    # per frame: "", "eager", "capture" or "replay"
        self._ba_events: Dict[int, tuple] = {}
        self._ba_seen = False
        # the map
        self.objects: Dict[int, sceneObject] = {}         # objects of the packed stack (the reference's obj_dict)
        self.scene_bg: Optional[sceneObject] = None
        self.optimiser = None
        self.ens = self.loop = None
        self.tracker: Optional[Tracker] = None
        self._tracked_set = None
        if not map:
            groups = tracker_groups(groups, cfg.do_bg, self.imap)
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
        the frame's pose when ``track=False`` (ignored otherwise).  In iMAP mode every pixel is instance 0 whatever
        ``inst`` holds (it may be None).  With ``assoc``, ``inst`` holds the raw ScanNet ids (instance + 1, as
        ``scannet.read_sequence`` yields them) and ``cls`` the classes.  Returns the frame index."""
        k, cfg, dev = self.k, self.cfg, self.device
        if self.imap:
            inst, cls = torch.zeros((cfg.W, cfg.H), dtype=torch.int32, device=dev), None
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
        if self.assoc is not None:
            visible = self._associate(slot, inst, depth, cls, pose)
            self._mark()
        if self.do_map:
            self._map_frame(slot, k, visible, pose)
        if self.ba_every:
            self.ba_frames.append([])
            self.ba_modes.append("")
            if self.objects and (k + 1) % self.ba_every == 0:
                self._bundle_adjust(k)
        store.release(slot)
        self._mark()
        self.k += 1
        return k

    def _associate(self, slot: int, inst, depth, cls, pose: torch.Tensor) -> Dict[int, torch.Tensor]:
        """ScanNet: the instance association at the frame's final pose (its only state change), then the slot and the
        store's tables relabelled from its output.  Returns the relabelled frame's kept labels and boxes."""
        store, dev = self.store, self.device
        inst = torch.as_tensor(inst).to(dev, torch.int32)
        max_id = int(inst.max()) + 1 if inst.numel() else 1          # as the loader sets it (ScanNet.associate)
        if max_id > store.max_id:
            raise _lib.VmbError(f"Slam: instance id {max_id - 1} does not fit the frame store's max_id={store.max_id}")
        labels, _ = self.assoc.frame(inst, torch.as_tensor(depth).to(dev, torch.float32),
                                     T=pose.cpu().numpy(), sem=cls, max_id=max_id)
        store.relabel(slot, labels, self.assoc.last_bbox)
        kb = torch.cat([store.stats[:, 7:8].float(), store.bbox], 1).cpu()
        return {int(i): kb[i, 1:] for i in torch.nonzero(kb[:, 0]).flatten().tolist()}

    def _mark(self, new_frame: bool = False) -> None:
        if self.timing:
            if new_frame:
                self.events.append([])
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.events[-1].append(e)

    def phase_times(self) -> dict:
        """With ``timing``: per frame, device milliseconds of ``ingest`` (with the keep-flag read), ``track``,
        ``assoc`` (only with ``assoc``: the association, the relabel and its table read), ``bookkeeping`` (keyframes,
        insertion, tables: host work the device waits for) and ``map``, ``ba`` (the bundle-adjustment pass with its
        table fill; 0.0 where none ran) and ``frame``."""
        torch.cuda.synchronize(self.device)
        phases = ("ingest", "track") + (("assoc",) if self.assoc is not None else ()) + ("bookkeeping", "map")
        out = {k: [] for k in phases + ("ba", "frame")}
        for k, ev in enumerate(self.events):
            d = [a.elapsed_time(b) for a, b in zip(ev[:-1], ev[1:])]
            if len(d) == len(phases) - 1:                  # no mapping mark (map=False, or no object yet)
                d = d + [0.0]
            ba = self._ba_events[k][0].elapsed_time(self._ba_events[k][1]) if k in self._ba_events else 0.0
            d[-1] -= ba                                    # the pass runs inside the last interval, after the map
            for key, v in zip(phases, d):
                out[key].append(v)
            out["ba"].append(ba)
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
        if self.ba is not None:
            self.ba.graph, self._ba_seen = None, False     # eager on the next pass, then captured again

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
        if self.joint is not None:
            self.loop.set_joint_tables(self.objects.values(), self.scene_bg)
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
                              kf_stride=cfg.keyframe_buffer_size, seed=self.seed, background=bg, joint=self.joint)
        if old is not None:
            self.loop.counter.copy_(old.counter)          # the sampler's draw counter runs on across re-stacks
        if self.do_track:
            self._rebuild_tracker()
        if self.ba_every:
            old = self.ba
            self.ba = BundleAdjuster(groups_from_objects(self._ba_objects().values()), cfg, self._ba_objects(),
                                     hold=0, **self.ba_kw)
            if old is not None:
                self.ba.counter.copy_(old.counter)        # the pass's draw counter runs on across re-stacks too
            self._ba_seen = False

    def _rebuild_tracker(self) -> None:
        objs = list(self.objects.values()) + ([self.scene_bg] if self.scene_bg is not None else [])
        groups = tracker_groups(groups_from_objects(objs), self.cfg.do_bg, self.imap)
        old = self.tracker
        self.tracker = Tracker(groups, self.cfg, **self.track_kw)
        if old is not None:
            self.tracker.counter.copy_(old.counter)        # the tracker's draw counter runs on too
        self._tracked_set = None
        self.mapped = {i for _, ids in groups for i in ids if i is not None}

    # ---- bundle adjustment -------------------------------------------------------------------------------------------
    def _ba_objects(self) -> Dict[int, sceneObject]:
        objs = dict(self.objects)
        if self.scene_bg is not None:
            objs[0] = self.scene_bg
        return objs

    def _bundle_adjust(self, k: int) -> None:
        """One pass after frame k's mapping frame: eager on the first pass of an object set, captured on the second,
        replayed after that (with ``graph``)."""
        ba, objs = self.ba, self._ba_objects()
        if self.timing:
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record()
        if not self.graph or not self._ba_seen:
            win = ba.run(self.store, self.poses, objs)
            self._ba_seen, mode = True, "eager"
        else:
            mode = "replay"
            if ba.graph is None or ba.pose_tables.cap != self.store.capacity:
                ba.capture(self.store, self.poses, objs)
                mode = "capture"
            win = ba.replay(self.store, self.poses, objs)
        if self.timing:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            self._ba_events[len(self.events) - 1] = (e0, e1)
        if win:
            self.ba_loss[k] = ba.losses[-1]
            self.ba_frames[-1] = list(win)
            self.ba_modes[-1] = mode

    # ---- the record --------------------------------------------------------------------------------------------------
    def result(self) -> dict:
        """The per-frame record read back (one copy at the end): ``poses`` [N, 4, 4] fp64, ``lost`` [N] bool,
        ``track_loss`` [N] fp64 (the tracker's last iteration; nan where not tracked), ``map_loss`` [N] (the last
        mapping iteration; nan where not mapped), ``tracked_ids``, ``inserted`` {object id: frame}, ``track_modes``,
        the frame store's final ``store_capacity``, ``ba_loss`` [N] fp64 (the last bundle-adjustment iteration's
        loss at frames where a pass ran; nan elsewhere), ``ba_frames`` (per frame, the frame ids its pass moved) and
        ``ba_modes``."""
        n = self.k
        ba_loss = self.ba_loss[:n].cpu().numpy() if self.ba_loss is not None else np.full(n, np.nan)
        return {"ba_loss": ba_loss, "ba_frames": [list(f) for f in self.ba_frames] or [[] for _ in range(n)],
                "ba_modes": list(self.ba_modes) or [""] * n,
                "poses": self.poses[:n].cpu().numpy(), "lost": self.lost[:n].cpu().numpy(),
                "track_loss": self.track_loss[:n].cpu().numpy(), "map_loss": self.map_loss[:n].cpu().numpy(),
                "tracked_ids": [list(i) for i in self.tracked_ids], "inserted": dict(self.inserted),
                "track_modes": list(self.track_modes), "store_capacity": self.store.capacity}
