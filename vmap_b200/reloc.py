"""Relocalise a frame against the object map on the GPU: the tracking loss of many candidate poses in one launch.

A ``Tracker`` is a local optimiser: started outside its basin it converges to a wrong pose and nothing catches it.
``Relocalizer`` re-acquires the pose from a coarse prior by scoring a deterministic spread of candidate poses around it
with K10's loss (``vmb_reloc_score``, ``csrc/k_reloc.cuh``: the fused hidden-32 tile, forward only, many hypotheses
per CTA) and keeping the best on the device (``vmb_reloc_select``).  Per call, with no host read:

    round 1   every prior x ``hypotheses(n_hyp, rot_deg, trans)``            -> scores -> top K
    round 2   every round-1 pose x the same set at a quarter of the spread    -> scores
    pick      the top K of each round and the caller's extra candidates (e.g. the tracker's own result), best first

The samples are the camera-frame points the tracker drew for the frame: slice 0 (its iteration 1), so the score of a
pose is, bit for bit, the loss ``Tracker.losses[0]`` reports from that pose when the tracker has one group.  Hidden-32
groups on ``impl="fused"`` only: scoring needs the fp16 weight image and has no K10 fallback.
"""
from __future__ import annotations

import ctypes as C
import math
from functools import lru_cache
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from .ensemble import _ptr, _stream

ROUND2_SHRINK = 0.25         # round 2 searches around each round-1 winner at this fraction of the spread


def _halton(i: int, base: int) -> float:
    f, r = 1.0, 0.0
    while i > 0:
        f /= base
        r += f * (i % base)
        i //= base
    return r


def _exp_so3(w: np.ndarray) -> np.ndarray:
    th = float(np.linalg.norm(w))
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + math.sin(th) / th * K + (1.0 - math.cos(th)) / th ** 2 * (K @ K)


@lru_cache(maxsize=32)
def _hypotheses(n: int, rot_deg: float, trans: float) -> np.ndarray:
    D = np.tile(np.eye(4), (n, 1, 1))
    ga = math.pi * (3.0 - math.sqrt(5.0))                  # golden angle
    for k in range(1, n):
        z = 1.0 - 2.0 * (k - 0.5) / max(n - 1, 1)         # rotation axis: Fibonacci sphere point k
        rr = math.sqrt(max(0.0, 1.0 - z * z))
        axis = np.array([rr * math.cos(ga * k), rr * math.sin(ga * k), z])
        D[k, :3, :3] = _exp_so3(axis * math.radians(rot_deg) * _halton(k, 2))
        u, v = _halton(k, 5), _halton(k, 7)                # translation: direction and radius from Halton
        zt = 1.0 - 2.0 * u
        rt = math.sqrt(max(0.0, 1.0 - zt * zt))
        d = np.array([rt * math.cos(2 * math.pi * v), rt * math.sin(2 * math.pi * v), zt])
        D[k, :3, 3] = d * trans * _halton(k, 3)
    D.setflags(write=False)
    return D


def hypotheses(n: int, rot_deg: float, trans: float) -> np.ndarray:
    """``n`` deterministic pose perturbations [n, 4, 4] fp64: the identity first, then rotations about Fibonacci-sphere
    axes by Halton angles in [0, rot_deg) and translations of Halton radius in [0, trans) along Halton directions.
    Applied on the right of a prior (``T @ D``), so rotations turn about the camera centre."""
    if n < 1 or not rot_deg >= 0.0 or not trans >= 0.0:
        raise ValueError("hypotheses: need n >= 1, rot_deg >= 0 and trans >= 0")
    return _hypotheses(int(n), float(rot_deg), float(trans))


def _compose(P: torch.Tensor, D: torch.Tensor) -> torch.Tensor:
    """[P, n, 4, 4] = P[p] @ D[j] in fp64 on the device, as elementwise products summed in a fixed order."""
    return (P[:, None, :, :, None] * D[None, :, None, :, :]).sum(-2)


class Relocalizer:
    """Pose hypotheses scored against the map's hidden-32 objects on the samples a ``Tracker`` drew for the frame.

    ``source``: a ``Tracker`` (``impl="fused"``) that has tracked or sampled the frame, whose live groups, sample
    buffers (slice 0) and status word are reused; or a list of tracking groups with their samples bound (e.g.
    ``SampleGroup(..., impl="fused")``), with a status word of its own.  ``n_hyp`` hypotheses per prior in round 1 and
    per round-1 winner in round 2, ``top_k`` winners kept, spread ``rot_deg`` degrees / ``trans`` metres."""

    def __init__(self, source, n_hyp: int = 256, top_k: int = 8, rot_deg: float = 30.0, trans: float = 0.3):
        if not 1 <= top_k <= min(n_hyp, _lib.RELOC_MAX_K):
            raise _lib.VmbError(f"Relocalizer: top_k must be in [1, min(n_hyp, {_lib.RELOC_MAX_K})]")
        if top_k * n_hyp > _lib.RELOC_MAX_HYP:
            raise _lib.VmbError(f"Relocalizer: top_k * n_hyp must be at most {_lib.RELOC_MAX_HYP}")
        if isinstance(source, (list, tuple)):
            self._fixed = list(source)
            self.device = self._fixed[0].ens.device
            self.status = torch.zeros(4, dtype=torch.int32, device=self.device)
        else:
            self._fixed, self.tracker = None, source
            self.device, self.status = source.device, source.status
        self.n_hyp, self.top_k = n_hyp, top_k
        self.D1 = torch.from_numpy(hypotheses(n_hyp, rot_deg, trans).copy()).to(self.device)
        self.D2 = torch.from_numpy(hypotheses(n_hyp, rot_deg * ROUND2_SHRINK, trans * ROUND2_SHRINK).copy()).to(self.device)

    def _groups(self):
        live = self._fixed if self._fixed is not None else self.tracker._live()
        for g in live:
            if g.path != "fused":
                raise _lib.VmbError("Relocalizer: scoring runs on hidden-32 groups on impl='fused' only "
                                    f"(a hidden-{g.ens.hidden} group takes path {g.path!r})")
        return live

    def _on_device(self, t) -> bool:
        dev = torch.device(self.device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        return torch.is_tensor(t) and t.device == dev

    def _poses(self, poses, who: str) -> torch.Tensor:
        if not self._on_device(poses) or not poses.is_floating_point() or poses.dim() not in (2, 3) \
                or tuple(poses.shape[-2:]) != (4, 4):
            raise _lib.VmbError(f"{who}: poses must be a floating-point [H, 4, 4] tensor on {self.device}")
        return poses.reshape(-1, 4, 4).to(torch.float64).contiguous()

    def score(self, poses: torch.Tensor, terms: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Slice-0 tracking loss [H] fp64 of each pose of ``poses`` [H, 4, 4] (device, fp64); ``terms``: optional
        [H, B, 4] contiguous fp64 device tensor of per-object terms (L_d, L_c, L_o, total), one group only (a second
        group's call would overwrite the first's rows).  Arguments are checked before any launch."""
        live = self._groups()
        poses = self._poses(poses, "Relocalizer.score")
        H = poses.shape[0]
        if not 1 <= H <= _lib.RELOC_MAX_HYP:
            raise _lib.VmbError(f"Relocalizer.score: 1 .. {_lib.RELOC_MAX_HYP} poses")
        if terms is not None:
            if len(live) != 1:
                raise _lib.VmbError(f"Relocalizer.score: terms need exactly one group ({len(live)} are live)")
            B = len(live[0].active)
            if not (self._on_device(terms) and terms.dtype == torch.float64 and tuple(terms.shape) == (H, B, 4)
                    and terms.is_contiguous()):
                raise _lib.VmbError(f"Relocalizer.score: terms must be a contiguous fp64 [{H}, {B}, 4] tensor on "
                                    f"{self.device}")
        scores = torch.zeros(H, dtype=torch.float64, device=poses.device)
        a = _lib.TrackArgs()
        a.n_groups, a.n_iter, a.iter = len(live), 1, 1
        a.colour_scaling, a.opacity_scaling = live[0].ens.colour_scaling, live[0].ens.opacity_scaling
        a.status = _ptr(self.status)
        for gi, g in enumerate(live):
            g.bind(a.group[gi], 0)
        for gi, g in enumerate(live):
            e = g.ens
            with e._on_device():
                _lib.check(e._handle, e.lib.vmb_reloc_score(e._handle, C.byref(a), gi, H, _ptr(poses), _ptr(scores),
                                                            _ptr(terms) if terms is not None else None, _ptr(e.image),
                                                            _stream()), "vmb_reloc_score")
        return scores

    def select(self, scores: torch.Tensor, poses: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """The ``k`` best (lowest score, ties to the lower index, non-finite last): (indices [k] int32, poses [k,4,4]).
        ``scores`` [n] and ``poses`` [n, 4, 4]: fp64 tensors on the groups' device; 1 <= k <= min(n, RELOC_MAX_K)."""
        if not (self._on_device(scores) and scores.dtype == torch.float64 and scores.dim() == 1):
            raise _lib.VmbError(f"Relocalizer.select: scores must be a 1-D fp64 tensor on {self.device}")
        n = scores.numel()
        if not 1 <= n <= _lib.RELOC_MAX_HYP:
            raise _lib.VmbError(f"Relocalizer.select: 1 .. {_lib.RELOC_MAX_HYP} scores")
        if not (self._on_device(poses) and poses.dtype == torch.float64 and tuple(poses.shape) == (n, 4, 4)):
            raise _lib.VmbError(f"Relocalizer.select: poses must be an fp64 [{n}, 4, 4] tensor on {self.device}")
        if not isinstance(k, (int, np.integer)) or isinstance(k, bool) or not 1 <= k <= min(n, _lib.RELOC_MAX_K):
            raise _lib.VmbError(f"Relocalizer.select: k must be in [1, min(n, {_lib.RELOC_MAX_K})]")
        k = int(k)
        scores = scores.contiguous()
        idx = torch.empty(k, dtype=torch.int32, device=scores.device)
        out = torch.empty(k, 4, 4, dtype=torch.float64, device=scores.device)
        e = self._groups()[0].ens
        poses = poses.contiguous()
        with e._on_device():
            _lib.check(e._handle, e.lib.vmb_reloc_select(e._handle, n, _ptr(scores), _ptr(poses), k, _ptr(idx),
                                                         _ptr(out), _stream()), "vmb_reloc_select")
        return idx, out

    def relocalise(self, priors: torch.Tensor, extra: Optional[torch.Tensor] = None):
        """Relocalise the tracker's frame from ``priors`` [P, 4, 4] (device fp64 T_wc), with the optional ``extra``
        candidates [E, 4, 4] scored alongside.  Returns (pose [4, 4], score [1], scores_topk [top_k]) device fp64
        tensors, best first; no host sync."""
        priors = priors.reshape(-1, 4, 4).to(torch.float64)
        if priors.shape[0] * self.n_hyp > _lib.RELOC_MAX_HYP:
            raise _lib.VmbError(f"Relocalizer: priors * n_hyp must be at most {_lib.RELOC_MAX_HYP}")
        K = self.top_k
        h1 = _compose(priors, self.D1).reshape(-1, 4, 4).contiguous()
        s1 = self.score(h1)
        i1, top1 = self.select(s1, h1, K)
        h2 = _compose(top1, self.D2).reshape(-1, 4, 4).contiguous()
        s2 = self.score(h2)
        i2, top2 = self.select(s2, h2, K)
        cands = [top1, top2]
        scores = [s1.index_select(0, i1.long()), s2.index_select(0, i2.long())]
        if extra is not None:
            ex = extra.reshape(-1, 4, 4).to(torch.float64).contiguous()
            cands.append(ex)
            scores.append(self.score(ex))
        cand, sc = torch.cat(cands), torch.cat(scores)
        idx, best = self.select(sc, cand, K)
        top = sc.index_select(0, idx.long())
        return best[0].clone(), top[:1].clone(), top
