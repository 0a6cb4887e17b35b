"""Host restatement of the project's Philox4x32-10 draws, bit for bit.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

The ray sampler (``vmap_b200/csrc/k_sampler.cuh``) and the surface sampler
(``vmap_b200/csrc/k_eval.cuh``) draw their randoms from Philox4x32-10 counters.
Philox is integer arithmetic, so the draws can be restated exactly on the host:

* ``philox4x32_10`` is the kernel's round loop, vectorised over numpy arrays
  (it reproduces the Random123 known-answer vectors);
* ``draw_randoms_philox`` returns the canonical per-ray arrays that
  ``sampler_oracle.sample_from_randoms`` consumes, drawn from the kernel's
  counter layout.  Every uniform is bitwise; the normals go through float32
  Box-Muller at the kernel's rounding points, where the kernel's ``logf`` /
  ``sincospif`` are 1-ulp functions, so a normal can differ from the kernel's
  in its last bit;
* ``surface_uniforms`` restates the surface sampler's stream.

Counter layout of the ray sampler, key (k0, k1) = (low, high 32 bits of seed),
counter (c0, c1, c2, c3) = (index, stream, object b of the launch, low 32 bits
of offset):

    stream 0   c0 = keyframe draw f      word 0      -> kf
    stream 1   c0 = ray i                words 0, 1  -> u_w, u_h
    stream 2   c0 = i * 8 + chunk c      words 0..3  -> u_z[4c .. 4c+3]
    stream 3   c0 = i * 8 + chunk c      words 0..3  -> normals 4c .. 4c+3

Surface sampler: counter (i mod 2^32, i >> 32, 4, 0), key = seed.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

import numpy as np
import torch

_M32 = np.uint64(0xFFFFFFFF)
_MUL0, _MUL1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_WEYL0, _WEYL1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_SHIFT32 = np.uint64(32)

STREAM_KF, STREAM_UV, STREAM_UZ, STREAM_NRM = 0, 1, 2, 3
SURFACE_STREAM = 4


def philox4x32_10(c0, c1, c2, c3, k0, k1) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Philox4x32-10 of counter (c0, c1, c2, c3) under key (k0, k1); arguments broadcast, results are uint32."""
    c0, c1, c2, c3, k0, k1 = (np.asarray(x).astype(np.uint64) & _M32 for x in (c0, c1, c2, c3, k0, k1))
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(c0, c1, c2, c3, k0, k1)
    for _ in range(10):
        p0, p1 = _MUL0 * c0, _MUL1 * c2                      # < 2^64: exact in uint64
        hi0, lo0 = p0 >> _SHIFT32, p0 & _M32
        hi1, lo1 = p1 >> _SHIFT32, p1 & _M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + _WEYL0) & _M32, (k1 + _WEYL1) & _M32
    return tuple(x.astype(np.uint32) for x in (c0, c1, c2, c3))


def u01(x) -> np.ndarray:
    """The kernel's uniform: the low 24 bits of a word times 2^-24, in float32 (exact)."""
    return (np.asarray(x, np.uint32) & np.uint32(0xFFFFFF)).astype(np.float32) * np.float32(2.0 ** -24)


def seed_key(seed: int) -> Tuple[int, int]:
    seed = int(seed) & (2 ** 64 - 1)
    return seed & 0xFFFFFFFF, seed >> 32


def _sincospi(x32: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """sin / cos of pi * x (x float32), rounded once to float32."""
    x = x32.astype(np.float64) * np.pi
    return np.sin(x).astype(np.float32), np.cos(x).astype(np.float32)


def _box_muller(q, sd: np.float32) -> np.ndarray:
    """[M, 4] float32 normals from four words per row, as the kernel forms them: sqrt(-2 log(1-u)) and sincospi(2u),
    one float32 rounding per operation (log rounded once from float64)."""
    one, m2, two = np.float32(1), np.float32(-2), np.float32(2)
    r = [np.sqrt(m2 * np.log((one - u01(q[k])).astype(np.float64)).astype(np.float32)) for k in (0, 2)]
    s0, c0 = _sincospi(two * u01(q[1]))
    s1, c1 = _sincospi(two * u01(q[3]))
    g = np.stack([r[0] * c0, r[0] * s0, r[1] * c1, r[1] * s1], axis=-1)
    return g * sd


def keyframe_draws(seed: int, offset: int, b: int, n_frames: int, n_kf: int, latest: Sequence[int],
                   stream: int = STREAM_KF, latest_from: int = 3) -> np.ndarray:
    """kf [n_frames] int64: the last two draws are ``latest`` when n_kf >= ``latest_from`` (the kernel: n_kf > 2);
    with n_frames == 1 that one draw is latest[1]."""
    k0, k1 = seed_key(seed)
    f = np.arange(n_frames, dtype=np.uint64)
    o = philox4x32_10(f, stream, b, offset, k0, k1)
    kf = np.minimum((u01(o[0]) * np.float32(n_kf)).astype(np.int64), n_kf - 1)
    if n_kf >= latest_from:
        for j in range(max(n_frames - 2, 0), n_frames):
            kf[j] = int(latest[j - (n_frames - 2)])
    return kf


def draw_randoms_philox(seed: int, offset: int, b: int, n_frames: int, n_pix: int, n_kf: int, latest: Sequence[int],
                        n1: int, n2: int, surface_eps: float, streams: Sequence[int] = (0, 1, 2, 3),
                        latest_from: int = 3) -> Dict[str, torch.Tensor]:
    """The canonical per-ray arrays (kf [F], u_w / u_h [F,P], u_z [N,S], nrm [N,n2]) object ``b`` of a launch draws
    in Philox mode.  ``streams`` (the c1 word of kf, u_w/u_h, u_z, normals) and ``latest_from`` are the layout's
    parameters; they default to the kernel's and exist so tests can build deliberately wrong schemes."""
    S = n1 + n2
    assert S <= 32 and n_frames * n_pix < 2 ** 29
    k0, k1 = seed_key(seed)
    N = n_frames * n_pix
    kf = keyframe_draws(seed, offset, b, n_frames, n_kf, latest, streams[0], latest_from)
    i = np.arange(N, dtype=np.uint64)
    o = philox4x32_10(i, streams[1], b, offset, k0, k1)
    u_w, u_h = u01(o[0]).reshape(n_frames, n_pix), u01(o[1]).reshape(n_frames, n_pix)
    u_z = np.empty((N, (S + 3) // 4 * 4), np.float32)
    for c in range((S + 3) // 4):
        q = philox4x32_10(i * np.uint64(8) + np.uint64(c), streams[2], b, offset, k0, k1)
        u_z[:, 4 * c:4 * c + 4] = np.stack([u01(w) for w in q], axis=-1)
    sd = np.float32(surface_eps) / np.float32(3.0)
    nrm = np.empty((N, (n2 + 3) // 4 * 4), np.float32)
    for c in range((n2 + 3) // 4):
        nrm[:, 4 * c:4 * c + 4] = _box_muller(philox4x32_10(i * np.uint64(8) + np.uint64(c), streams[3], b, offset,
                                                            k0, k1), sd)
    t = torch.from_numpy
    return {"kf": t(kf), "u_w": t(u_w), "u_h": t(u_h), "u_z": t(np.ascontiguousarray(u_z[:, :S])),
            "nrm": t(np.ascontiguousarray(nrm[:, :n2]))}


def sampler_counters(b: int, offset: int, n_frames: int, n_pix: int, n1: int, n2: int) -> np.ndarray:
    """[M, 4] uint32: every Philox counter object ``b`` of a launch may use (normals counted for every ray)."""
    N, S = n_frames * n_pix, n1 + n2
    i = np.arange(N, dtype=np.int64)
    parts = [np.stack([np.arange(n_frames), np.zeros(n_frames, np.int64)], -1),
             np.stack([i, np.ones(N, np.int64)], -1)]
    for stream, n in ((STREAM_UZ, S), (STREAM_NRM, n2)):
        c0 = (i[:, None] * 8 + np.arange((n + 3) // 4)[None, :]).reshape(-1)
        parts.append(np.stack([c0, np.full(c0.shape, stream)], -1))
    c01 = np.concatenate(parts)
    assert (c01[:, 0] < 2 ** 32).all()
    return np.concatenate([c01, np.full((len(c01), 1), b), np.full((len(c01), 1), int(offset) & 0xFFFFFFFF)],
                          axis=1).astype(np.uint32)


def surface_counters(n: int) -> np.ndarray:
    """[n, 4] uint32: the surface sampler's counters (i mod 2^32, i >> 32, 4, 0)."""
    i = np.arange(n, dtype=np.uint64)
    return np.stack([i & _M32, i >> _SHIFT32, np.full(n, SURFACE_STREAM, np.uint64), np.zeros(n, np.uint64)],
                    -1).astype(np.uint32)


def surface_uniforms(seed: int, n: int) -> np.ndarray:
    """[n, 3] float64 (u0, u1, u2) of ``vmb_surface_sample``'s seeded mode: a 53-bit u0, 32-bit u1 / u2."""
    k0, k1 = seed_key(seed)
    c = surface_counters(n)
    o = philox4x32_10(c[:, 0], c[:, 1], c[:, 2], c[:, 3], k0, k1)
    u0 = ((o[0] >> np.uint32(5)).astype(np.float64) * 67108864.0 + (o[1] >> np.uint32(6)).astype(np.float64)) \
        * (1.0 / 9007199254740992.0)
    return np.stack([u0, o[2].astype(np.float64) / 4294967296.0, o[3].astype(np.float64) / 4294967296.0], axis=-1)


def sample_philox(objects, n_frames: int, n_pix: int, rays_dir: torch.Tensor, cfg, seed: int, offset: int,
                  b_index: Sequence[int] = None, **layout) -> Dict[str, torch.Tensor]:
    """What one Philox-mode sampler launch over ``objects`` returns, in ``BatchedSampler.sample``'s layout (pcs
    [B,N,S,3], z [B,N,S], gt_depth [B,N], gt_colour [B,N,3], gt_rgb_u8 [B,N,3], sem [B,N], mask_depth [B,N]).
    ``objects``: (rgbs_batch, depth_batch, t_wc_batch, bbox, n_kf, latest) per object, CPU tensors.  ``b_index``
    replaces each object's counter word c2 (default: its position) and ``layout`` goes to ``draw_randoms_philox``."""
    from . import sampler_oracle as so
    n1, n2 = cfg.n_bins_cam2surface, cfg.n_bins
    N = n_frames * n_pix
    keys = ("gt_rgb_u8", "gt_depth", "mask_depth", "sem", "pcs", "z")
    outs = {k: [] for k in keys}
    for b, (rgbs, depth, twc, bbox, n_kf, latest) in enumerate(objects):
        cb = b if b_index is None else b_index[b]
        rnd = draw_randoms_philox(seed, offset, cb, n_frames, n_pix, n_kf, latest, n1, n2, cfg.surface_eps, **layout)
        res = so.sample_from_randoms(rnd, rgbs, depth, twc, bbox, rays_dir, cfg)
        for k, v in zip(keys, res):
            outs[k].append(v)
    out = {"pcs": torch.stack(outs["pcs"]).reshape(-1, N, n1 + n2, 3),
           "z": torch.stack(outs["z"]).reshape(-1, N, n1 + n2),
           "gt_depth": torch.stack(outs["gt_depth"]).reshape(-1, N),
           "gt_rgb_u8": torch.stack(outs["gt_rgb_u8"]).reshape(-1, N, 3),
           "sem": torch.stack(outs["sem"]).reshape(-1, N),
           "mask_depth": torch.stack(outs["mask_depth"]).reshape(-1, N)}
    out["gt_colour"] = out["gt_rgb_u8"].float() / 255.0          # train.py:257 (fp32 division, as the kernel)
    return out
