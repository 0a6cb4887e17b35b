"""One mapping frame as ONE CUDA graph: batched sampler (K3) + the frame's optimisation steps (K0+K1+K2 each).

The reference's per-frame loop (train.py:195-326) is launch-bound at its shipped configuration (20 objects x 120
rays per step: ~25 us of kernel work per step behind ~60 us of Python + launches).  ``FrameLoop`` captures

    K3 pass 1 -> K3 pass 2 [-> the same two passes for the background model] -> draw counter += 1
      -> n_iter x [ fused step on the it-th ray slice (+ AdamW) [-> background step + AdamW] -> loss ]

once, on persistent buffers, and replays it per frame; the one small host->device copy of the per-frame tables is
enqueued right before the replay (outside the graph, so the pinned source buffer is guarded by its own event and
the host can fill the next frame's tables as soon as that copy -- not the whole frame -- has completed).  What changes between frames lives in device memory (Adam
step counter, sampler draw counter) or in the pinned table buffer (keyframe slots / boxes / counts), so a replay
draws fresh samples and continues the optimiser exactly as the eager loop would.

Joint mode (``joint=JointPoses(...)``): the keyframe poses are optimised with the weights.  The sampler draws the same
Philox samples in the camera frame and records each draw's keyframe; per iteration, for a hidden-64/128/256 stack (iMAP)

    vmb_joint_step_lw (world points from each draw's pose, the mapping step, per-ray pose rows from its embedding
      gradient) -> vmb_adam (weights) -> vmb_ba_update (one Adam + Exp over the window of keyframe poses)

and for a hidden-32 stack (vMAP), with the ``Background`` model as the update's second group when there is one,

    vmb_joint_step_fused (the same, on the fused step, AdamW inside it) [-> vmb_joint_step_lw on the background
      -> its vmb_adam] -> vmb_ba_update (one Adam + Exp over the window of both groups' keyframe poses)

and after the last iteration the refined poses go in fp32 to the store's slots (and to the background's keyframe copies).
The iteration's loss is the mapping loss (plus the background's).  Frame 0 (the anchor) never moves; the pose Adam
moments restart with every frame, as a bundle-adjustment pass's do.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import _lib
from .ba import PoseTables, _BaGroup, ba_args, ba_update, fill_kf_frame
from .ensemble import VmapEnsemble
from .sampler import BatchedSampler, KeyframeSet, KeyframeTables, SamplerTables
from .utils import capture_graph


class Background:
    """The separate background model of a ``do_bg`` run (train.py:147-152): a 1-object ensemble (hidden 128 in the shipped
    config) with its own sampler (5 + 9 bins), its own keyframe buffers and its own ray budget
    (``n_iter_per_frame * win_size_bg`` draws of ``n_samples_per_frame_bg`` pixels, train.py:196-199)."""

    def __init__(self, ens: VmapEnsemble, sampler: BatchedSampler, n_frames: int, n_pix: int):
        assert ens.n_obj == 1
        self.ens, self.smp, self.n_frames, self.n_pix = ens, sampler, n_frames, n_pix
        self.tables = SamplerTables(ens.device, 1)
        self.out = sampler._outputs(1, n_frames * n_pix, sampler.n1 + sampler.n2, False)


class JointPoses:
    """The opt-in joint mode of ``FrameLoop``: ``poses`` is the fp64 pose table [F, 4, 4] (row = frame id) whose keyframe
    rows every mapping iteration moves with the weights, at rates ``lr_rot`` / ``lr_trans``; ``hold`` (the anchor frame)
    never moves."""

    def __init__(self, poses: torch.Tensor, lr_rot: float, lr_trans: float, hold: int = 0):
        assert poses.dtype == torch.float64 and poses.dim() == 3 and poses.shape[1:] == (4, 4) and poses.is_contiguous()
        self.poses, self.lr_rot, self.lr_trans, self.hold = poses, lr_rot, lr_trans, hold


class _JointGroup(_BaGroup):
    """The mapping stack as the one group of the joint step: FrameLoop's sample buffers, bound per iteration the way a
    bundle-adjustment group is (``_BaGroup.bind``): ``n_pix`` rays of ``win`` draws of ``n_pix_draw`` pixels."""

    def __init__(self, ens: VmapEnsemble, out, kf_out: torch.Tensor, n_pix: int, n_pix_draw: int, KF: int):
        self.ens, self.out, self.kf_out, self.lw = ens, out, kf_out, True
        self.n_pix, self.n_pix_draw, self.S, self.KF = n_pix, n_pix_draw, out["pcs"].shape[2], KF
        self.win, self.n_draws = n_pix // n_pix_draw, kf_out.shape[1]
        self.rows_dev = torch.arange(ens.n_obj, dtype=torch.int32, device=ens.device)
        self._alloc_rows(ens.n_obj)


class FrameLoop:
    def __init__(self, ens: VmapEnsemble, sampler: BatchedSampler, n_frames: int, n_pix: int, n_iter: int,
                 rays_dir: torch.Tensor, store=None, kf_stride: int = 0, seed: int = 0, first_offset: int = 0,
                 background: Optional[Background] = None, joint: Optional[JointPoses] = None):
        """``n_frames * n_pix`` rays are drawn per object per frame and consumed in ``n_iter`` slices
        (train.py:198,270-277).  ``store``/``kf_stride``: shared keyframe store mode (keyframes.FrameStore).
        ``background``: the ``do_bg`` model, sampled and stepped inside the same graph; its loss is added to the
        iteration's loss as train.py:308-316 does (`batch_loss += bg_loss`).  ``joint``: optimise the keyframe poses
        with the weights (see the module docstring); needs the store and whole draws per iteration, and a background
        only with a hidden-32 stack (its keyframe copies hold up to ``kf_stride`` keyframes).  Its tables come from
        ``set_joint_tables``."""
        assert (n_frames * n_pix) % n_iter == 0, "rays per frame must split evenly over the iterations"
        self.ens, self.smp, self.store = ens, sampler, store
        self.bg = background
        if background is not None:
            assert (background.n_frames * background.n_pix) % n_iter == 0
            assert background.ens.device == ens.device
        self.n_frames, self.n_pix, self.n_iter = n_frames, n_pix, n_iter
        self.rays_dir = rays_dir.contiguous()
        self.seed = seed
        dev = ens.device
        B = ens.n_obj
        self.tables = SamplerTables(dev, B, kf_stride=kf_stride if store is not None else 0)
        self.out = sampler._outputs(B, n_frames * n_pix, sampler.n1 + sampler.n2, False)
        self.counter = torch.full((1,), first_offset, dtype=torch.int64, device=dev)     # sampler draw counter
        self.losses = torch.zeros(n_iter, dtype=torch.float32, device=dev)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.joint = joint
        if joint is not None:
            if store is None or ens.image is None:
                raise ValueError("FrameLoop: joint poses need the frame store and the ensemble's fp16 image")
            if background is not None and (ens.hidden != 32 or background.ens.image is None
                                           or background.ens.hidden == 32):
                raise ValueError("FrameLoop: joint poses with a background model need a hidden-32 stack and a "
                                 "hidden-64/128/256 background")
            assert n_frames % n_iter == 0, "joint poses: every iteration takes whole draws"
            self.kf_out = torch.zeros(B, n_frames, dtype=torch.int32, device=dev)
            self.jg = _JointGroup(ens, self.out, self.kf_out, n_frames * n_pix // n_iter, n_pix, kf_stride)
            groups, shapes = [self.jg], [(B, kf_stride)]
            if background is not None:
                assert background.n_frames % n_iter == 0, "joint poses: every iteration takes whole background draws"
                self.bg_kf_out = torch.zeros(1, background.n_frames, dtype=torch.int32, device=dev)
                self.jbg = _JointGroup(background.ens, background.out, self.bg_kf_out,
                                       background.n_frames * background.n_pix // n_iter, background.n_pix, kf_stride)
                self.bg_loss = torch.zeros(1, dtype=torch.float32, device=dev)
                self.bg_t_wc = None             # the background's keyframe copies (set_joint_tables)
                groups.append(self.jbg)
                shapes.append((1, kf_stride))
            self.max_win = min(_lib.BA_MAX_WIN, sum(b * kf for b, kf in shapes))
            self.pose_tables = PoseTables(dev, shapes, self.max_win, kf_stride if background is not None else 0)
            f64 = dict(dtype=torch.float64, device=dev)
            self.pose_adam = torch.zeros(self.max_win, 12, **f64)
            self.pose_scratch = torch.zeros(8 * sum(g.ens.n_obj * g.win for g in groups) + 6 * self.max_win, **f64)
            self.pose_status = torch.zeros(4, dtype=torch.int32, device=dev)

    # ---- per-frame host work: only the small tables ------------------------------------------------------
    def set_objects(self, sets: Sequence[KeyframeSet]) -> None:
        self.tables.fill_objects(sets)

    def set_store_tables(self, kt: KeyframeTables) -> None:
        self.tables.fill_store(kt)

    def set_background(self, kf: KeyframeSet) -> None:
        self.bg.tables.fill_objects([kf])

    def set_joint_tables(self, objects, background=None) -> List[int]:
        """Joint mode: the frame id of every keyframe of ``objects`` (the stack's sceneObjects, row order) and, with a
        background model, of ``background`` (its sceneObject, whose keyframe copies ``t_wc_batch`` receive the refined
        poses), and the window of poses this frame moves; returns the window.  A store that grew since the capture, or
        a background whose copies moved, drops the graph."""
        pt = self.pose_tables
        if pt.layout(self.store):
            self.graph = None                       # the captured frame points at the old tables
            self.jg.kf_frame = pt.kf_frame(0)
            if self.bg is not None:
                self.jbg.kf_frame = pt.kf_frame(1)
        fills = [lambda t: fill_kf_frame(list(objects), self.store, t)]
        if self.bg is not None:
            fills.append(lambda t: fill_kf_frame([background], self.store, t, bg=True))
            if self.bg_t_wc is not background.t_wc_batch:
                self.bg_t_wc, self.graph = background.t_wc_batch, None
        return pt.prepare(self.store, fills, self.joint.hold, 1 if self.bg is not None else None)

    # ---- the frame -----------------------------------------------------------------------------------------
    def _enqueue(self, upload: bool = True) -> None:
        s, R = self.smp, self.n_frames * self.n_pix // self.n_iter
        bg = self.bg
        if upload:
            self.tables.upload()
            if bg is not None:
                bg.tables.upload()
        joint = self.joint is not None
        if bg is not None:      # train.py:196-206: the background draws its own rays (same draw counter, its own stream key)
            kw = dict(camera_frame=True, kf_out=self.bg_kf_out) if joint else {}
            bg.smp.sample(None, bg.n_frames, bg.n_pix, self.rays_dir, seed=self.seed + 0x5bd1e995,
                          tables=bg.tables, out=bg.out, offset_dev=self.counter, **kw)
            Rb = bg.n_frames * bg.n_pix // self.n_iter
        if joint:
            if upload:
                self.pose_tables.upload()
            s.sample_store(self.store, self.tables, self.n_frames, self.n_pix, self.rays_dir, seed=self.seed,
                           out=self.out, offset_dev=self.counter, camera_frame=True, kf_out=self.kf_out)
            self.counter += 1
            self._joint_iterations(R, Rb if bg is not None else 0)
            return
        if self.store is not None:
            s.sample_store(self.store, self.tables, self.n_frames, self.n_pix, self.rays_dir, seed=self.seed,
                           out=self.out, offset_dev=self.counter)
        else:
            s.sample(None, self.n_frames, self.n_pix, self.rays_dir, seed=self.seed,
                     tables=self.tables, out=self.out, offset_dev=self.counter)
        self.counter += 1
        for it in range(self.n_iter):
            self.ens.step({k: v[:, it * R:(it + 1) * R] for k, v in self.out.items()}, loss_out=self.losses[it:it + 1])
            if bg is not None:  # train.py:308-316
                self.losses[it] += bg.ens.step({k: v[:, it * Rb:(it + 1) * Rb] for k, v in bg.out.items()})

    def _joint_iterations(self, R: int, Rb: int) -> None:
        j, pt, g, bg = self.joint, self.pose_tables, self.jg, self.bg
        groups = [g] + ([self.jbg] if bg is not None else [])
        targets = [(pt.frame_of, self.store.t_wc, self.store.capacity)]
        if bg is not None:
            targets.append((pt.bg_frame_of, self.bg_t_wc, pt.bg_kf))
        a = ba_args(groups, self.n_iter, j.poses, pt.window_dev, self.max_win, j.hold, self.pose_adam,
                    self.pose_scratch, j.lr_rot, j.lr_trans, None, self.pose_status, targets=targets)
        for it in range(self.n_iter):
            a.iter = it + 1
            for gi, gr in enumerate(groups):
                gr.bind(a.group[gi], it)
            batch = {k: v[:, it * R:(it + 1) * R] for k, v in self.out.items()}
            if self.ens.hidden == 32:       # AdamW inside the fused step
                self.ens.joint_step_fused(batch, a, 0, loss_out=self.losses[it:it + 1])
            else:
                self.ens.joint_step(batch, a, 0, loss_out=self.losses[it:it + 1])
                self.ens.adam_step()
            if bg is not None:              # train.py:308-316: the background's loss joins the iteration's
                bg.ens.joint_step({k: v[:, it * Rb:(it + 1) * Rb] for k, v in bg.out.items()}, a, 1,
                                  loss_out=self.bg_loss)
                bg.ens.adam_step()
                self.losses[it] += self.bg_loss[0]
            ba_update(self.ens, a)

    def run_eager(self) -> torch.Tensor:
        """The same frame without a graph (reference for tests / first frames)."""
        self.ens.poll_status()
        self._enqueue()
        return self.losses

    def capture(self) -> None:
        """Warm up once (kernel attributes, allocator) on a side stream, then capture.  The warm-up frame and the
        capture itself do not advance the optimiser or the draw counter."""
        all_ens = [self.ens] + ([self.bg.ens] if self.bg is not None else [])
        keep = [t for e in all_ens for t in (e.params, e.grads, e.exp_avg, e.exp_avg_sq, e.step_counter)]
        keep += [e.image for e in all_ens if e.image is not None] + [self.counter]
        if self.joint is not None:
            keep += [self.joint.poses, self.store.t_wc] + ([self.bg_t_wc] if self.bg is not None else [])
        counts = [e.step_count for e in all_ens]
        self.graph = capture_graph(self.ens.device, self._enqueue, keep)
        for e, cn in zip(all_ens, counts):
            e.step_count = cn

    def run(self) -> torch.Tensor:
        """Replay the captured frame; returns the per-iteration summed losses (device tensor [n_iter])."""
        if self.graph is None:
            self.capture()
        self.ens.poll_status()            # raises LossExplode if an earlier frame tripped the device guard
        self.tables.upload()
        if self.joint is not None:
            self.pose_tables.upload()
        if self.bg is not None:
            self.bg.ens.poll_status()
            self.bg.tables.upload()
            self.bg.ens.step_count += self.n_iter
        self.graph.replay()
        self.ens.step_count += self.n_iter
        return self.losses
