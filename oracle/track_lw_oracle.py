"""fp16-faithful restatement (torch, fp64) of the layer-wise tracking step (``vmap_b200/csrc/k_track_lw.cuh``).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

The tracking rule is K10's (``oracle/track_oracle.py``) and, with a pose per ray, K11's (``oracle/ba_oracle.py``): the
loss of every object with the per-object, per-term empty-mask rule, var detached, the left-perturbation tangent.  The
network runs as ``oracle/lw_oracle.py`` runs the layer-wise training step, and this module rounds to fp16 exactly
where the tracking path stores fp16 (switches in ``lw_oracle.Rounding``; ``dh`` is unused, the path has no head
weight gradients):

- the embedding rows E at the posed point p / scale,
- the weights, read from the fp16 image (biases and both heads stay fp32),
- every forward activation, ``relu(half_sat(acc + bias))``,
- ``dYc = half(clamp(gate(hc > 0) * (2^8 dh_c @ W_oc), +-60000))``,
- the gated dgrads ``dY4 .. dY1 = half_sat(acc (+ 2^8 dh_a * w_a)) * (x_prev > 0)``.

Everything else is fp64: the render, loss and head gradients (the kernel: fp64 render and loss, fp32 head gradients),
the embedding gradient dE and the pose terms.  With ``ROUND_OFF`` the gradient is the exact fp64 gradient of
``track_oracle`` (``tests/test_track_lw_oracle.py``).

The L1 losses make the gradient depend on the sign of each ray's residual; a ray whose residual lies inside the fp16
noise of the forward could take different signs here and in the kernel.  ``signs`` [B,R,5] overrides them.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch

from .lw_oracle import DH_CLAMP, INV_LS, LS, ROUND_ALL, ROUND_OFF, Rounding, _half  # noqa: F401
from .vmap_oracle import N_DIRS, PE_KEY


def evaluate(params: Dict[str, torch.Tensor], scale, batch: Dict[str, torch.Tensor], poses, frames=None,
             rounding: Rounding = ROUND_ALL, cs: float = 5.0, os_: float = 10.0, signs: Optional[torch.Tensor] = None,
             var: Optional[torch.Tensor] = None) -> dict:
    """One tracking step of a stack of B objects.

    params: stacked ``[B, *shape]`` fp32 master weights; scale: scalar or [B]; batch: pcs [B,R,S,3] camera-frame
    points q, z, gt_depth, gt_colour, sem, mask_depth; poses: [F,4,4] (or one [4,4]) camera-to-world; frames: [B,R]
    pose index of each ray (default 0; -1 = no pose: the ray contributes nothing, the counts still include it);
    var: [B,R] rendered variance to weight the depth term with (default: this render's, detached).

    Returns a dict of fp64 tensors: ``rows`` [B,R,6] each ray's pose terms ((R q) x g, g) summed over its samples,
    ``ray_terms`` [B,R,3] each ray's (L_d, L_c, L_o) share, ``terms`` [B,4] per-object loss terms and weighted total,
    ``grad`` [F,6] the per-pose tangent gradient, ``loss`` the scalar loss, ``var`` [B,R] the rendered variance,
    and before the fp16 clamp: ``dyc_pre`` [B,P,H] the gated, loss-scaled dYc and ``rank1`` [B,P,H] dY4's loss-scaled
    d_alpha w_a term (the values the kernel counts into status[1])."""
    f64 = dict(dtype=torch.float64)
    rnd = rounding
    p = {k: v.to(**f64) for k, v in params.items()}
    W_in, W_m1, W_cat, W_m2, W_cl = (_half(p[k + ".weight"], rnd.weights)
                                     for k in ("in_layer.0", "mid1.0.0", "cat_layer.0", "mid2.0.0", "color_linear.0"))
    w_a, W_oc = p["out_alpha.weight"][:, 0], p["out_color.weight"]
    q = batch["pcs"].to(**f64)
    B, R, S, _ = q.shape
    H = W_m1.shape[-1]
    P = R * S
    sc = torch.as_tensor(scale, **f64).expand(B).reshape(B, 1, 1)
    T = torch.as_tensor(np.asarray(poses, np.float64)).reshape(-1, 4, 4)
    fr_idx = torch.zeros(B, R, dtype=torch.int64) if frames is None else torch.as_tensor(frames, dtype=torch.int64)
    ok = fr_idx >= 0
    f = fr_idx.clamp(min=0)
    Rr, tr_ = T[f, :3, :3], T[f, :3, 3]                                                  # [B,R,3,3], [B,R,3]
    rq = torch.einsum("brij,brsj->brsi", Rr, q)                                         # R q
    pw = rq + tr_[:, :, None, :]
    mm = torch.matmul
    tr = lambda x: x.transpose(1, 2)                                                     # noqa: E731

    # ---- embedding at the pose (k_tlw_pe) ----
    t = pw.reshape(B, P, 3) / sc
    dirs = p[PE_KEY]
    proj = mm(t, tr(dirs))
    ang = [proj * (math.pi * 2.0 ** k) for k in range(6)]
    band = torch.cat([torch.sin(a) for a in ang], -1)
    emb1 = _half(torch.cat([t, band[..., :4 * N_DIRS]], -1), rnd.emb)
    emb2 = _half(band[..., 4 * N_DIRS:], rnd.emb)

    # ---- forward GEMMs ----
    def layer(acc, bias):
        return torch.relu(_half(acc + p[bias][:, None, :], rnd.acts))
    X1 = layer(mm(emb1, tr(W_in)), "in_layer.0.bias")
    X2 = layer(mm(X1, tr(W_m1)), "mid1.0.0.bias")
    X3 = layer(mm(X2, tr(W_cat[..., :H])) + mm(emb1, tr(W_cat[..., H:])), "cat_layer.0.bias")
    X4 = layer(mm(X3, tr(W_m2)), "mid2.0.0.bias")
    XC = layer(mm(X4, tr(W_cl[..., :H])) + mm(emb2, tr(W_cl[..., H:])), "color_linear.0.bias")

    # ---- heads + render + loss (k_tlw_render: K10's rule) ----
    alpha = (10.0 * (mm(X4, w_a[..., None])[..., 0] + p["out_alpha.bias"])).reshape(B, R, S)
    col = torch.sigmoid(mm(XC, tr(W_oc)) + p["out_color.bias"][:, None, :]).reshape(B, R, S, 3)
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
    cnt = torch.stack([(md & (sem != 0)).sum(1), (sem != 0).sum(1), (sem != 2).sum(1)], 1)   # all rays of the slice
    inv = torch.where(cnt > 0, 1.0 / (cnt.double() + 1e-10), torch.zeros_like(cnt, dtype=torch.float64))
    m_o = ((sem != 0) & ok).double()
    m_s = ((sem != 2) & ok).double()
    m_d = md.double() * m_o
    info = 1.0 / (torch.sqrt(Vw) + 1e-4)
    e_d = D - batch["gt_depth"].to(**f64)
    e_c = C - batch["gt_colour"].to(**f64)
    e_o = O - m_o
    ray_terms = torch.stack([e_d.abs() * m_d * info * inv[:, :1], e_c.abs().sum(-1) * m_o * inv[:, 1:2],
                             e_o.abs() * m_s * inv[:, 2:3]], -1)                       # [B,R,3]
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
    dh_a = (10.0 * docc * oc * fr).reshape(B, P)
    dh_c = (gC[..., None, :] * w[..., None] * col * (1.0 - col)).reshape(B, P, 3)
    dyc_pre = (XC > 0) * mm(LS * dh_c, W_oc)                                            # before the +-60000 clamp
    dYc = _half(dyc_pre, rnd.dyc, DH_CLAMP)

    # ---- backward to the embedding only ----
    def gate(acc, x_prev):
        return _half(acc, rnd.dgrad) * (x_prev > 0)
    rank1 = (LS * dh_a)[..., None] * w_a[:, None, :]                                      # dY4's d_alpha term
    dY4 = gate(mm(dYc, W_cl[..., :H]) + rank1, X4)
    dY3 = gate(mm(dY4, W_m2), X3)
    dY2 = gate(mm(dY3, W_cat[..., :H]), X2)
    dY1 = gate(mm(dY2, W_m1), X1)
    dE1 = mm(dY3, W_cat[..., H:]) + mm(dY1, W_in)
    dE2 = mm(dYc, W_cl[..., H:])

    # ---- pose terms (k_tlw_pose) and rows ----
    dband = torch.cat([dE1[..., 3:], dE2], -1)
    dproj = sum(dband[..., k * N_DIRS:(k + 1) * N_DIRS] * torch.cos(ang[k]) * (math.pi * 2.0 ** k) for k in range(6))
    dt = INV_LS * (dE1[..., :3] + mm(dproj, dirs))                                      # d loss / d t  [B,P,3]
    g = (dt / sc).reshape(B, R, S, 3)
    pt = torch.cat([torch.cross(rq, g, dim=-1), g], -1) * ok[..., None, None]            # [B,R,S,6]
    rows = pt.sum(2)
    grad = torch.zeros(T.shape[0], 6, **f64)
    grad.index_add_(0, f.reshape(-1), rows.reshape(-1, 6))
    return {"rows": rows, "ray_terms": ray_terms, "terms": terms, "grad": grad, "loss": float(terms[:, 3].sum()),
            "var": V, "abs_sum": pt.abs().sum((1, 2)), "dyc_pre": dyc_pre, "rank1": rank1}
