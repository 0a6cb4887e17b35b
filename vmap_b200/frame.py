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
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

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


class FrameLoop:
    def __init__(self, ens: VmapEnsemble, sampler: BatchedSampler, n_frames: int, n_pix: int, n_iter: int,
                 rays_dir: torch.Tensor, store=None, kf_stride: int = 0, seed: int = 0, first_offset: int = 0,
                 background: Optional[Background] = None):
        """``n_frames * n_pix`` rays are drawn per object per frame and consumed in ``n_iter`` slices
        (train.py:198,270-277).  ``store``/``kf_stride``: shared keyframe store mode (keyframes.FrameStore).
        ``background``: the ``do_bg`` model, sampled and stepped inside the same graph; its loss is added to the
        iteration's loss as train.py:308-316 does (`batch_loss += bg_loss`)."""
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

    # ---- per-frame host work: only the small tables ------------------------------------------------------
    def set_objects(self, sets: Sequence[KeyframeSet]) -> None:
        self.tables.fill_objects(sets)

    def set_store_tables(self, kt: KeyframeTables) -> None:
        self.tables.fill_store(kt)

    def set_background(self, kf: KeyframeSet) -> None:
        self.bg.tables.fill_objects([kf])

    # ---- the frame -----------------------------------------------------------------------------------------
    def _enqueue(self, upload: bool = True) -> None:
        s, R = self.smp, self.n_frames * self.n_pix // self.n_iter
        bg = self.bg
        if upload:
            self.tables.upload()
            if bg is not None:
                bg.tables.upload()
        if bg is not None:      # train.py:196-206: the background draws its own rays (same draw counter, its own stream key)
            bg.smp.sample(None, bg.n_frames, bg.n_pix, self.rays_dir, seed=self.seed + 0x5bd1e995,
                          tables=bg.tables, out=bg.out, offset_dev=self.counter)
            Rb = bg.n_frames * bg.n_pix // self.n_iter
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
        if self.bg is not None:
            self.bg.ens.poll_status()
            self.bg.tables.upload()
            self.bg.ens.step_count += self.n_iter
        self.graph.replay()
        self.ens.step_count += self.n_iter
        return self.losses
