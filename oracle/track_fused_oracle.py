"""fp16-faithful restatement (torch, fp64) of the fused hidden-32 tracking step (``vmap_b200/csrc/k_track_fused.cuh``).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

Two restatements combined, neither copied:

- the network and its rounding points are ``oracle/fused_oracle.py``'s (the fused training step's tile: fp16 embedding,
  fp16 image weights and heads, fp16 activations, the fp16 dhead row feeding ``dYc`` and the alpha term of ``dY4``,
  the gated fp16 dgrads, the PE backward's fp32 cos ladder), with the ``Rounding`` switches of that module;
- the tracking rule is ``oracle/track_lw_oracle.py``'s (K10's and K11's): render in fp64 with ``1 - occ`` as
  ``sigmoid(-alpha)``, the per-object, per-term empty-mask rule, the loss scale applied at the head gradients, which are
  clamped to +-60000 (``DH_CLAMP``) before their fp16 pack, and the pose terms ``((R q) x g, g)`` in fp64.

The points are ``pose_point``'s (``k_track.cuh``): ``p = R q + t`` in fp32 from an fp32 copy of the fp64 pose, the fma
order ``fma(T2, qz, fma(T1, qy, T0 * qx)) + T3``, then ``p / scale`` in fp32 (``posed_points``; with ``proj32`` off the
fp64 points).  ``emb=`` takes the kernel's own embedding (``tests/test_fused_faithful_gpu.probe_embedding``) and
``signs=`` the L1 residual signs, as ``fused_oracle.fused_step`` does.  With ``ROUND_OFF`` the result is the exact fp64
gradient of ``oracle/track_oracle.py`` (``tests/test_track_fused_oracle.py``).
"""
from __future__ import annotations

import math
from dataclasses import replace
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import fused_oracle as fo
from .lw_oracle import DH_CLAMP, HALF_MAX, INV_LS, LS, _half
from .vmap_oracle import N_DIRS, PE_KEY

# the fused tracking step's roundings: fused_oracle's, with no dB (dproj, t16) and the head gradients clamped at 60000
ROUND_ALL = replace(fo.ROUND_ALL, dproj=False, t16=False, dh_lim=DH_CLAMP)
ROUND_OFF = fo.ROUND_OFF
Rounding = fo.Rounding


def _pose_table(poses) -> torch.Tensor:
    return torch.as_tensor(np.asarray(poses.cpu() if torch.is_tensor(poses) else poses, np.float64)).reshape(-1, 4, 4)


def posed_points(poses, frames, q: torch.Tensor, scale, fp32: bool = True):
    """(t [B,R,S,3], R q [B,R,S,3]) in fp64: the network input of each camera-frame point q [B,R,S,3] at the pose of its
    ray (``frames`` [B,R], default 0; -1 = no pose: t = 0) and the fp64 ``R q`` of the pose terms.  ``fp32``:
    ``pose_point``'s fp32 arithmetic, bit for bit; otherwise ``(R q + t) / scale`` in fp64."""
    T = _pose_table(poses)
    q = q.to(torch.float64)
    B, R = q.shape[:2]
    fr = torch.zeros(B, R, dtype=torch.int64) if frames is None else torch.as_tensor(frames, dtype=torch.int64)
    ok = (fr >= 0)[..., None, None]
    Tf = T[fr.clamp(min=0)]                                                             # [B,R,4,4]
    rq = torch.einsum("brij,brsj->brsi", Tf[..., :3, :3], q)
    sc = torch.as_tensor(scale, dtype=torch.float64).expand(B).reshape(B, 1, 1, 1)
    if not fp32:
        t = (rq + Tf[:, :, None, :3, 3]) / sc
    else:
        T32 = fo._f32(Tf)[:, :, None]                                                   # [B,R,1,4,4]
        x = fo._f32(T32[..., :3, 0] * fo._f32(q[..., 0:1]))
        x = fo._fma32(T32[..., :3, 1], fo._f32(q[..., 1:2]), x)
        x = fo._fma32(T32[..., :3, 2], fo._f32(q[..., 2:3]), x)
        x = fo._f32(x + T32[..., :3, 3])
        t = fo._f32(x / fo._f32(sc))
    return torch.where(ok, t, torch.zeros_like(t)), rq


def evaluate(params: Dict[str, torch.Tensor], scale, batch: Dict[str, torch.Tensor], poses, frames=None,
             rounding: Rounding = ROUND_ALL, cs: float = 5.0, os_: float = 10.0, signs: Optional[torch.Tensor] = None,
             var: Optional[torch.Tensor] = None, emb: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> dict:
    """One tracking step of a stack of B hidden-32 objects, as ``track_lw_oracle.evaluate`` describes its arguments and
    results (rows [B,R,6], ray_terms [B,R,3], terms [B,4], grad [F,6], loss, var), plus ``t`` [B,R,S,3] the network
    inputs.  emb: (E1 [B,R*S,87], E2 [B,R*S,42]) in the reference column order, the embedding to use."""
    f64 = dict(dtype=torch.float64)
    rnd = rounding
    p = {k: v.to(**f64) for k, v in params.items()}
    q = batch["pcs"].to(**f64)
    B, R, S, _ = q.shape
    P = R * S
    sc = torch.as_tensor(scale, **f64).expand(B).reshape(B, 1, 1)
    T = _pose_table(poses)
    fr_idx = torch.zeros(B, R, dtype=torch.int64) if frames is None else torch.as_tensor(frames, dtype=torch.int64)
    ok = fr_idx >= 0
    f = fr_idx.clamp(min=0)
    t, rq = posed_points(T, fr_idx, q, scale, rnd.proj32)
    mm, tr = torch.matmul, (lambda x: x.transpose(1, 2))

    # ---- E0 and the six forward stages (fused_oracle) ----
    dirs = p[PE_KEY]
    _, proj = fo.projections(t.reshape(B, P, 3), dirs, 1.0, rnd.proj32)               # scale 1: t as given
    if emb is None:
        band = fo.sin_bands(proj)
        emb1 = _half(torch.cat([t.reshape(B, P, 3), band[..., :4 * N_DIRS]], -1), rnd.emb)
        emb2 = _half(band[..., 4 * N_DIRS:], rnd.emb)
    else:
        emb1, emb2 = emb[0].to(**f64), emb[1].to(**f64)
    W, w_a, W_oc = fo._weights(p, rnd)
    H = W["mid1.0.0"].shape[-1]
    X1, X2, X3, X4, XC, raw_a, raw_c = fo._mlp(p, W, w_a, W_oc, emb1, emb2, rnd)

    # ---- render + loss (track_lw_oracle: K10's rule) ----
    alpha = raw_a.reshape(B, R, S)
    col = torch.sigmoid(raw_c).reshape(B, R, S, 3)
    oc, fr = torch.sigmoid(alpha), torch.sigmoid(-alpha)                                # fr = 1 - occ
    z = batch["z"].to(**f64)
    om = fr + 1e-10
    Tr = torch.cat([torch.ones_like(om[..., :1]), torch.cumprod(om, -1)[..., :-1]], -1)
    w = oc * Tr
    D, O = (w * z).sum(-1), w.sum(-1)
    C = (w[..., None] * col).sum(-2)
    V = (w * (z - D[..., None]) ** 2).sum(-1)
    Vw = V if var is None else var.to(**f64)
    sem, md = batch["sem"], batch["mask_depth"].bool()
    cnt = torch.stack([(md & (sem != 0)).sum(1), (sem != 0).sum(1), (sem != 2).sum(1)], 1)
    inv = torch.where(cnt > 0, 1.0 / (cnt.double() + 1e-10), torch.zeros_like(cnt, dtype=torch.float64))
    m_o = ((sem != 0) & ok).double()
    m_s = ((sem != 2) & ok).double()
    m_d = md.double() * m_o
    info = 1.0 / (torch.sqrt(Vw) + 1e-4)
    e_d = D - batch["gt_depth"].to(**f64)
    e_c = C - batch["gt_colour"].to(**f64)
    e_o = O - m_o
    ray_terms = torch.stack([e_d.abs() * m_d * info * inv[:, :1], e_c.abs().sum(-1) * m_o * inv[:, 1:2],
                             e_o.abs() * m_s * inv[:, 2:3]], -1)
    lt = ray_terms.sum(1)
    terms = torch.cat([lt, (lt[:, 0] + cs * lt[:, 1] + os_ * lt[:, 2])[:, None]], 1)
    sg = torch.cat([e_d[..., None], e_c, e_o[..., None]], -1).sign() if signs is None else signs.to(**f64)
    gD = sg[..., 0] * m_d * info * inv[:, :1]
    gC = (cs * m_o * inv[:, 1:2])[..., None] * sg[..., 1:4]
    gO = os_ * sg[..., 4] * m_s * inv[:, 2:3]
    Gs = gD[..., None] * z + (gC[..., None, :] * col).sum(-1) + gO[..., None]
    gw = Gs * w
    suffix = gw.flip(-1).cumsum(-1).flip(-1) - gw
    docc = Gs * Tr - suffix / om
    dh = LS * torch.cat([(10.0 * docc * oc * fr).reshape(B, P, 1),
                         (gC[..., None, :] * w[..., None] * col * (1.0 - col)).reshape(B, P, 3)], -1)
    dh16 = _half(dh, rnd.dh, rnd.dh_lim)                                                # clamp, fp16 dhead row
    feed = dh16 if rnd.dh_feeds else dh

    # ---- the input-gradient chain (fused_oracle's gates and rounding points) ----
    def gate(acc, x_prev, on_):
        return _half(acc, on_, HALF_MAX) * (x_prev > 0)
    W_cl, W_cat = W["color_linear.0"], W["cat_layer.0"]
    dYc = gate(mm(feed[..., 1:], W_oc), XC, rnd.dyc)
    dY4 = gate(mm(dYc, W_cl[..., :H]) + feed[..., :1] * w_a[:, None, :], X4, rnd.dgrad)
    dY3 = gate(mm(dY4, W["mid2.0.0"]), X3, rnd.dgrad)
    dY2 = gate(mm(dY3, W_cat[..., :H]), X2, rnd.dgrad)
    dY1 = gate(mm(dY2, W["mid1.0.0"]), X1, rnd.dgrad)
    dE1 = mm(dY3, W_cat[..., H:]) + mm(dY1, W["in_layer.0"])
    dE2 = mm(dYc, W_cl[..., H:])

    # ---- PE backward, pose terms and rows ----
    dband = torch.cat([dE1[..., 3:], dE2], -1)
    cb = fo.cos_bands(proj, rnd.cos32)
    pi = fo.PI_F if rnd.cos32 else math.pi
    dproj = sum(dband[..., k * N_DIRS:(k + 1) * N_DIRS] * (2.0 ** k) * cb[k] for k in range(fo.N_BANDS)) * pi
    dt = INV_LS * (dE1[..., :3] + mm(dproj, dirs))
    g = (dt / sc).reshape(B, R, S, 3)
    pt = torch.cat([torch.cross(rq, g, dim=-1), g], -1) * ok[..., None, None]
    rows = pt.sum(2)
    grad = torch.zeros(T.shape[0], 6, **f64)
    grad.index_add_(0, f.reshape(-1), rows.reshape(-1, 6))
    return {"rows": rows, "ray_terms": ray_terms, "terms": terms, "grad": grad, "loss": float(terms[:, 3].sum()),
            "var": V, "abs_sum": pt.abs().sum((1, 2)), "t": t}
