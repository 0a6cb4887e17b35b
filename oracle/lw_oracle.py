"""fp16-faithful restatement (torch, fp64) of the layer-wise step of the wide models (hidden 64 / 128 / 256).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

``vmap_b200/csrc/k_layerwise.cuh`` runs one object's step as wgmma GEMMs over all points with fp16 operands and
fp32 accumulation, plus thin CUDA-core kernels for the embedding, the heads + render + loss, the bias column sums
and the PE backward.  This module computes the same step in fp64 and rounds to fp16 exactly where the kernel
stores fp16 (``step_object`` and the epilogues of ``k_gemm_umma.cuh``):

- the embedding rows E (xyz/scale, the sin bands; the constant-1 bias columns are exact),
- the weights, read from the fp16 image (biases and both heads' weights stay fp32),
- every forward layer, ``relu(acc + bias)`` with a saturating fp16 pack,
- the head gradients ``dh16 = half(clamp(2^8 dh, +-60000))`` that feed the head weight gradients
  (the rank-1 term of the colour-layer dgrad and the head biases use the unrounded dh),
- the colour hidden gradient ``dYc = half(clamp(gate(hc > 0) * (2^8 dh_c @ W_oc), +-60000))``,
- the gated dgrads ``dY4 .. dY1 = half_sat(acc (+ 2^8 dh_a * w_a)) * (x_prev > 0)``.

The embedding gradient dE, the weight gradients ``2^-8 dY^T X`` and the PE backward are fp32 in the kernel and
exact here.  Each rounding point has a switch (``Rounding``); with ``ROUND_OFF`` the result is the exact fp64
gradient of ``oracle.vmap_oracle``'s model (checked by ``tests/test_lw_oracle.py``).

The L1 losses make the gradient depend on the sign of each ray's residual.  A ray whose residual lies inside the
fp16 noise of the forward can take different signs here and in the kernel, and that one ray then dominates any
comparison, so ``signs`` can override them: ``signs_from_render`` takes them from the kernel's own render outputs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from .vmap_oracle import ALL_KEYS, N_DIRS, PE_KEY

LS = 256.0                # loss scale of the fp16 gradients (common.cuh: LS)
INV_LS = 1.0 / LS
DH_CLAMP = 60000.0        # clamp of the scaled head gradients before their fp16 pack
HALF_MAX = 65504.0        # cvt.rn.satfinite.f16: saturate to the largest finite half


@dataclass(frozen=True)
class Rounding:
    """Which fp16 stores of the kernel are emulated."""
    emb: bool = True        # embedding rows E
    weights: bool = True    # GEMM weights from the fp16 image
    acts: bool = True       # forward activations X1..X4, XC
    dh: bool = True         # dh16, the B operand of the head weight-gradient GEMMs
    dyc: bool = True        # dYc, the colour hidden gradient written by the render kernel
    dgrad: bool = True      # dY4, dY3, dY2, dY1 of the gated dgrad GEMMs


ROUND_ALL = Rounding()
ROUND_OFF = Rounding(False, False, False, False, False, False)


def _half(x: torch.Tensor, on: bool, lim: float = HALF_MAX) -> torch.Tensor:
    return x.clamp(-lim, lim).half().to(x.dtype) if on else x


def mask_counts(sem: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """[B,4] int32 as k_mask_counts: depth rays, object rays, rays outside the 'other object' label, (unused)."""
    m_o = sem != 0
    out = torch.zeros(sem.shape[0], 4, dtype=torch.int32, device=sem.device)
    out[:, 0] = (m_o & mask.bool()).sum(1)
    out[:, 1] = m_o.sum(1)
    out[:, 2] = (sem != 2).sum(1)
    return out


def signs_from_render(depth, colour, opacity, batch) -> torch.Tensor:
    """[B,R,5] signs of the L1 residuals (depth, colour r, g, b, opacity) of a render, e.g. the kernel's own."""
    sem = batch["sem"]
    e_d = depth.double() - batch["gt_depth"].double()
    e_c = colour.double() - batch["gt_colour"].double()
    e_o = opacity.double() - (sem != 0).double()
    return torch.cat([e_d[..., None], e_c, e_o[..., None]], -1).sign()


def lw_step(params: Dict[str, torch.Tensor], scale, batch: Dict[str, torch.Tensor], counts: Optional[torch.Tensor] = None,
            signs: Optional[torch.Tensor] = None, rounding: Rounding = ROUND_ALL, colour_scaling: float = 5.0,
            opacity_scaling: float = 10.0, device=None):
    """One layer-wise step of a stack of objects.

    params: stacked ``[B, *shape]`` tensors keyed by ``vmap_oracle.ALL_KEYS`` (the fp32 master weights);
    scale: scalar or [B]; batch: the six step inputs; counts: [B,4] mask counts (default: from this batch -- pass
    the full batch's counts to run a sub-batch as part of it); signs: optional [B,R,5] residual signs.
    Returns ``(render, loss_terms, grads)``: render = (depth [B,R], var [B,R], colour [B,R,3], opacity [B,R]),
    loss_terms [B,4] = (L_depth, L_colour, L_opacity, weighted total), grads = {key: [B, *shape]}; all fp64."""
    dev = torch.device(device) if device is not None else batch["pcs"].device
    f64 = dict(dtype=torch.float64, device=dev)
    rnd = rounding
    p = {k: v.to(**f64) for k, v in params.items()}
    W_in, W_m1, W_cat, W_m2, W_cl = (_half(p[k + ".weight"], rnd.weights)
                                     for k in ("in_layer.0", "mid1.0.0", "cat_layer.0", "mid2.0.0", "color_linear.0"))
    w_a, W_oc = p["out_alpha.weight"][:, 0], p["out_color.weight"]                    # [B,H], [B,3,H] fp32
    pcs = batch["pcs"].to(**f64)
    B, R, S, _ = pcs.shape
    H = W_m1.shape[-1]
    P = R * S
    sc = torch.as_tensor(scale, **f64).expand(B).reshape(B, 1, 1)
    mm = torch.matmul
    tr = lambda x: x.transpose(1, 2)                                                  # noqa: E731

    # ---- embedding (k_lw_pe) ----
    t = pcs.reshape(B, P, 3) / sc
    dirs = p[PE_KEY]                                                                   # [B,21,3]
    proj = mm(t, tr(dirs))                                                             # [B,P,21]
    ang = [proj * (math.pi * 2.0 ** k) for k in range(6)]
    band = torch.cat([torch.sin(a) for a in ang], -1)                                  # frequency-major
    emb1 = _half(torch.cat([t, band[..., :4 * N_DIRS]], -1), rnd.emb)                 # [B,P,87]
    emb2 = _half(band[..., 4 * N_DIRS:], rnd.emb)                                      # [B,P,42]

    # ---- forward GEMMs (EPI_RELU_F16) ----
    def layer(acc, bias):
        return torch.relu(_half(acc + p[bias][:, None, :], rnd.acts))
    X1 = layer(mm(emb1, tr(W_in)), "in_layer.0.bias")
    X2 = layer(mm(X1, tr(W_m1)), "mid1.0.0.bias")
    X3 = layer(mm(X2, tr(W_cat[..., :H])) + mm(emb1, tr(W_cat[..., H:])), "cat_layer.0.bias")
    X4 = layer(mm(X3, tr(W_m2)), "mid2.0.0.bias")
    XC = layer(mm(X4, tr(W_cl[..., :H])) + mm(emb2, tr(W_cl[..., H:])), "color_linear.0.bias")

    # ---- heads + render + loss + head gradients (k_lw_heads_render) ----
    raw_a = mm(X4, w_a[..., None])[..., 0] + p["out_alpha.bias"]                       # [B,P]
    raw_c = mm(XC, tr(W_oc)) + p["out_color.bias"][:, None, :]                         # [B,P,3]
    oc = torch.sigmoid(raw_a * 10.0).reshape(B, R, S)
    col = torch.sigmoid(raw_c).reshape(B, R, S, 3)
    z = batch["z"].to(**f64)
    om = 1.0 - oc + 1e-10
    T = torch.cat([torch.ones_like(om[..., :1]), torch.cumprod(om, -1)[..., :-1]], -1)
    w = oc * T
    D = (w * z).sum(-1)
    O = w.sum(-1)
    C = (w[..., None] * col).sum(-2)
    V = (w * (z - D[..., None]) ** 2).sum(-1)

    sem = batch["sem"].to(dev)
    mask = batch["mask_depth"].to(dev)
    cnt = mask_counts(sem, mask) if counts is None else counts.to(dev)
    on = (cnt[:, :3] != 0).all(0).double()                                             # whole-batch early-out
    inv = 1.0 / (cnt[:, :3].float() + 1e-10).double()                                  # fp32 in the kernel
    m_o = (sem != 0).double()
    m_s = (sem != 2).double()
    m_d = mask.bool().double() * m_o
    info = 1.0 / (torch.sqrt(V) + 1e-4)
    e_d = D - batch["gt_depth"].to(**f64)
    e_c = C - batch["gt_colour"].to(**f64)
    e_o = O - m_o
    l_d = on[0] * (e_d.abs() * m_d * info).sum(1) * inv[:, 0]
    l_c = on[1] * (e_c.abs().sum(-1) * m_o).sum(1) * inv[:, 1]
    l_o = on[2] * (e_o.abs() * m_s).sum(1) * inv[:, 2]
    loss_terms = torch.stack([l_d, l_c, l_o, l_d + colour_scaling * l_c + opacity_scaling * l_o], 1)
    sg = torch.cat([e_d[..., None], e_c, e_o[..., None]], -1).sign() if signs is None else signs.to(**f64)

    gD = on[0] * sg[..., 0] * m_d * info * inv[:, :1]                                  # [B,R]
    gC = (on[1] * colour_scaling * m_o * inv[:, 1:2])[..., None] * sg[..., 1:4]        # [B,R,3]
    gO = on[2] * opacity_scaling * sg[..., 4] * m_s * inv[:, 2:3]
    Gs = gD[..., None] * z + (gC[..., None, :] * col).sum(-1) + gO[..., None]         # d loss / d w  [B,R,S]
    gw = Gs * w
    suffix = gw.flip(-1).cumsum(-1).flip(-1) - gw                                     # sum over later samples
    docc = Gs * T - suffix / om
    dh_a = (10.0 * docc * oc * (1.0 - oc)).reshape(B, P)
    dh_c = (gC[..., None, :] * w[..., None] * col * (1.0 - col)).reshape(B, P, 3)
    dh = torch.cat([dh_a[..., None], dh_c], -1)                                        # [B,P,4] fp32 in the kernel
    dh16 = _half(LS * dh, rnd.dh, DH_CLAMP)
    dYc = _half((XC > 0) * mm(LS * dh_c, W_oc), rnd.dyc, DH_CLAMP)

    g = {}
    g["out_alpha.weight"] = INV_LS * mm(tr(dh16[..., :1]), X4)
    g["out_alpha.bias"] = dh_a.sum(1, keepdim=True)
    g["out_color.weight"] = INV_LS * mm(tr(dh16[..., 1:]), XC)
    g["out_color.bias"] = dh_c.sum(1)

    # ---- gated dgrads (EPI_GATE_F16) and weight gradients (EPI_ATOMIC, k_lw_colsum) ----
    def gate(acc, x_prev):
        return _half(acc, rnd.dgrad) * (x_prev > 0)

    def wgrad(dY, X, key):
        g[key + ".weight"] = INV_LS * mm(tr(dY), X)
        g[key + ".bias"] = INV_LS * dY.sum(1)

    dY4 = gate(mm(dYc, W_cl[..., :H]) + (LS * dh_a)[..., None] * w_a[:, None, :], X4)
    wgrad(dYc, torch.cat([X4, emb2], -1), "color_linear.0")
    dE2 = mm(dYc, W_cl[..., H:])
    dY3 = gate(mm(dY4, W_m2), X3)
    wgrad(dY4, X3, "mid2.0.0")
    dY2 = gate(mm(dY3, W_cat[..., :H]), X2)
    wgrad(dY3, torch.cat([X2, emb1], -1), "cat_layer.0")
    dY1 = gate(mm(dY2, W_m1), X1)
    wgrad(dY2, X1, "mid1.0.0")
    wgrad(dY1, emb1, "in_layer.0")
    dE1 = mm(dY3, W_cat[..., H:]) + mm(dY1, W_in)

    # ---- PE backward (k_lw_pe_bwd) ----
    dband = torch.cat([dE1[..., 3:], dE2], -1)                                         # [B,P,126] frequency-major
    dproj = sum(dband[..., k * N_DIRS:(k + 1) * N_DIRS] * torch.cos(ang[k]) * (math.pi * 2.0 ** k) for k in range(6))
    g[PE_KEY] = INV_LS * mm(tr(dproj), t)

    render = (D, V, C, O)
    return render, loss_terms, {k: g[k].reshape(params[k].shape) for k in ALL_KEYS}
