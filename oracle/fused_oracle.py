"""fp16-faithful restatement (torch, fp64) of the fused hidden-32 step (``k_step_fused``, ``impl="umma"``).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

``vmap_b200/csrc/k_step_fused.cuh`` runs the whole step of a hidden-32 object in one kernel: wgmma on fp16 operands
with fp32 accumulation, the heads, the volume render and the losses in fp32 registers.  This module computes the same
step in fp64 and rounds where that kernel rounds.  Each rounding point has a switch (``Rounding``); the kernel lines
each one restates:

- ``emb``: the embedding E1 / E2 as fp16 (E0 block: ``pack_h2`` of the MUFU sin / cos pair and the angle-doubling
  ladder of ``k_umma_image.cuh``).  By default the caller passes the kernel's own embedding (``emb=``, read back through
  ``eval_points``); otherwise the bands are fp16 of fp64 sin.  The constant-1 columns are exact.
- ``proj32``: ``t = x * fp32(1 / scale)`` and the projections in fp32 in ``um::project4``'s fma order
  ``fma(bz, t2, fma(by, t1, bx * t0))`` (the direction-20 ``sin_ladder`` / ``cos_ladder`` argument has the same order).
- ``weights``: the hidden-layer weights from the fp16 image (``k_umma_image.cuh`` ``umma_fill_image_index``); biases
  and the PE directions stay fp32.
- ``heads``: both head weight matrices from the fp16 image (``IMG_WA16``, ``IMG_WOC16``).
- ``acts``: ``relu(satfinite(acc + bias))`` for fc1..fc4 and hc (``epi_relu``, ``pack_relu_h2``).
- ``dh``: ``dh16 = satfinite(LS * dh)``.  The loss scale is applied at the loss gradient (``gD``, ``kc``, ``gO``), so
  the fp32 chain from there to ``dh`` carries it; the dhead row is packed with ``cvt.rn.satfinite`` (65504).
- ``dh_feeds``: dh16, not the unrounded ``LS * dh``, feeds ``dYc`` (``d_hc = dhead @ W_oc``), the alpha term of ``dY4``
  (``dhead @ W_a``) and the head bias gradients (emb2's constant-1 column of the heads wgrad).
- ``dyc`` / ``dgrad``: ``dYc``, then ``dY4 .. dY1`` as ``satfinite(acc) * (x_prev > 0)`` (``epi_dgrad``).
- weight and bias gradients ``INV_LS * dY16^T X16``: exact here; the kernel sums them in fp32 wgmma accumulators and
  its per-CTA partial rows in fp32.  The embedding gradient dE is fp32 in the kernel and exact here.
- ``cos32``: the PE backward's cos ladder in fp32 (``cos4_x2`` / ``cos_doubling4_x2`` / ``cos_ladder``): the seed
  ``cos(pi r)`` correctly rounded to fp32, then ``c_{k+1} = fma(2 c_k, c_k, -1)`` in fp32, and ``dproj`` scaled by
  fp32(pi).  Off: fp64 cos.
- ``dproj``: ``dproj16``, the fp16 A operand of the dB wgrad (the ``FG_DPR`` block).
- ``t16``: dB multiplies dproj16 by the fp16 ``t`` columns of E1 (``dB = INV_LS * dproj16^T t16``).

Inputs the kernel decides per ray are taken as given: ``signs`` overrides the L1 residual signs (``signs_from_render``
takes them from the kernel's own render: a residual inside the fp16 noise may flip, and that one ray would dominate
any comparison), ``var`` the ray variances behind the depth-loss weight (the kernel's fp32 variance cancels on rays
whose weight sits on one sample, and 1 / (sqrt(var) + 1e-4) amplifies that) and ``counts`` the mask counts (a sub-batch run with the full batch's counts is part of that batch).
The kernel pads each tile with points whose occupancy is forced to 0 and whose dhead row stays zero, so they add
nothing to any sum; the dense [B, R, S] arrays here have no padding.

``LW_PLACEMENT`` moves the rounding points to where the layer-wise path (``oracle/lw_oracle.py``) has them; with it the
result equals ``lw_step`` at hidden 32 (checked by ``tests/test_fused_oracle.py``), so the two restatements differ only
in the places listed above.  With ``ROUND_OFF`` it is the exact fp64 gradient of ``oracle.vmap_oracle``'s model.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace
from typing import Dict, Optional, Tuple

import torch

from .lw_oracle import DH_CLAMP, HALF_MAX, INV_LS, LS, _half, mask_counts, signs_from_render  # noqa: F401
from .vmap_oracle import ALL_KEYS, N_DIRS, PE_KEY

PI_F = 3.14159274101257324        # float32(pi), VMB_PI_F
N_BANDS = 6


@dataclass(frozen=True)
class Rounding:
    """Which roundings of the fused kernel are emulated (see the module docstring for the kernel lines)."""
    emb: bool = True
    proj32: bool = True
    weights: bool = True
    heads: bool = True
    acts: bool = True
    dh: bool = True
    dh_feeds: bool = True
    dyc: bool = True
    dgrad: bool = True
    cos32: bool = True
    dproj: bool = True
    t16: bool = True
    dh_lim: float = HALF_MAX      # saturation of dh16 and dYc (the layer-wise path clamps at 60000)


ROUND_ALL = Rounding()
ROUND_OFF = Rounding(*([False] * 12))
LW_PLACEMENT = Rounding(proj32=False, heads=False, dh_feeds=False, cos32=False, dproj=False, t16=False,
                        dh_lim=DH_CLAMP)
SWITCHES = ("emb", "proj32", "weights", "heads", "acts", "dh", "dh_feeds", "dyc", "dgrad", "cos32", "dproj", "t16")


def flipped(name: str, base: Rounding = ROUND_ALL) -> Rounding:
    """``base`` with one switch inverted."""
    return replace(base, **{name: not getattr(base, name)})


def saturation_batch(B: int, R: int, S: int, seed: int = 0, spread: float = 1e-3):
    """A batch built to push the loss-scaled head gradient up: one depth ray per object and each ray's samples within
    ``spread`` of its depth, so the depth-loss weight 1 / (sqrt(var) + 1e-4) / n_depth is large."""
    b = synthetic(B, R, S, seed)
    g = torch.Generator().manual_seed(seed + 1)
    d = b["gt_depth"].clamp_min(0.5)
    b["gt_depth"] = d.contiguous()
    b["z"] = (d[..., None] + (torch.rand(B, R, S, generator=g) - 0.5) * spread).sort(-1).values.contiguous()
    b["mask_depth"] = torch.zeros(B, R, dtype=torch.bool)
    b["mask_depth"][:, 0] = True
    b["sem"][:, 0] = 1
    return b


def synthetic(B, R, S, seed):
    from .vmap_oracle import synthetic_batch
    if S > 1:
        return synthetic_batch(B, R, S, seed=seed, n_cam2surf=min(5, S - 1))
    b = synthetic_batch(B, R, 2, seed=seed, n_cam2surf=1)
    b["pcs"], b["z"] = b["pcs"][:, :, :1].contiguous(), b["z"][:, :, :1].contiguous()
    return b


def _f32(x: torch.Tensor) -> torch.Tensor:
    return x.float().double()


def _fma32(a, b, c):
    """fp32 fma restated in fp64: the product of two fp32 values is exact in fp64, one rounding to fp32 after the sum
    (a double rounding is possible but needs the fp64 sum to land on an fp32 tie)."""
    return _f32(a * b + c)


def projections(pcs: torch.Tensor, dirs: torch.Tensor, scale, fp32: bool = True):
    """(t [B,P,3], proj [B,P,21]) in fp64.  ``fp32``: the kernel's fp32 arithmetic (E0 block, ``um::project4``):
    ``t = x * fp32(1 / scale)``, ``proj = fma(bz, t2, fma(by, t1, bx * t0))``; otherwise ``pcs / scale`` and the fp64
    matrix product."""
    B = pcs.shape[0]
    x = pcs.reshape(B, -1, 3)
    dev = x.device
    sc = torch.as_tensor(scale, dtype=torch.float64, device=dev).expand(B)
    if not fp32:
        t = x.double() / sc.reshape(B, 1, 1)
        return t, torch.matmul(t, dirs.double().transpose(1, 2))
    isc = _f32(1.0 / sc.float().double()).reshape(B, 1, 1)               # 1.0f / scale: correctly rounded
    t = _f32(x.float().double() * isc)
    d = dirs.float().double()                                             # [B,21,3]
    p = _f32(t[..., 0:1] * d[:, None, :, 0])
    p = _fma32(t[..., 1:2], d[:, None, :, 1], p)
    p = _fma32(t[..., 2:3], d[:, None, :, 2], p)
    return t, p


def _reduce(proj):
    """r = proj - 2 rint(proj / 2): exact in fp32, and sin / cos(pi 2^k r) = sin / cos(pi 2^k proj)."""
    return proj - 2.0 * torch.round(0.5 * proj)


def sin_bands(proj):
    """[B,P,126] frequency-major sin(pi 2^k proj) in fp64 (k = 0..5)."""
    r = _reduce(proj)
    return torch.cat([torch.sin(r * (math.pi * 2.0 ** k)) for k in range(N_BANDS)], -1)


def cos_bands(proj, fp32: bool = True):
    """[6][B,P,21] cos(pi 2^k proj): the kernel's fp32 ladder, or fp64 cos."""
    r = _reduce(proj)
    if not fp32:
        return [torch.cos(r * (math.pi * 2.0 ** k)) for k in range(N_BANDS)]
    c = [_f32(torch.cos(math.pi * r))]
    for _ in range(1, N_BANDS):
        c.append(_fma32(c[-1] + c[-1], c[-1], -1.0))
    return c


def embedding(pcs, dirs, scale, rounding: Rounding = ROUND_ALL):
    """(E1 [B,P,87], E2 [B,P,42]) in the reference column order: fp16 of fp64 sin of the (fp32) projection."""
    t, proj = projections(pcs, dirs, scale, rounding.proj32)
    band = sin_bands(proj)
    e1 = _half(torch.cat([t, band[..., :4 * N_DIRS]], -1), rounding.emb)
    e2 = _half(band[..., 4 * N_DIRS:], rounding.emb)
    return e1, e2


def _weights(p, rnd: Rounding):
    W = {k: _half(p[k + ".weight"], rnd.weights) for k in ("in_layer.0", "mid1.0.0", "cat_layer.0", "mid2.0.0",
                                                          "color_linear.0")}
    w_a = _half(p["out_alpha.weight"][:, 0], rnd.heads)                                 # [B,H]
    W_oc = _half(p["out_color.weight"], rnd.heads)                                      # [B,3,H]
    return W, w_a, W_oc


def _mlp(p, W, w_a, W_oc, emb1, emb2, rnd: Rounding):
    """Forward layers and heads: (X1, X2, X3, X4, XC, raw alpha (x10) [B,P], raw colour [B,P,3])."""
    mm, tr = torch.matmul, (lambda x: x.transpose(1, 2))
    H = W["mid1.0.0"].shape[-1]

    def layer(acc, bias):
        return torch.relu(_half(acc + p[bias][:, None, :], rnd.acts))
    X1 = layer(mm(emb1, tr(W["in_layer.0"])), "in_layer.0.bias")
    X2 = layer(mm(X1, tr(W["mid1.0.0"])), "mid1.0.0.bias")
    X3 = layer(mm(X2, tr(W["cat_layer.0"][..., :H])) + mm(emb1, tr(W["cat_layer.0"][..., H:])), "cat_layer.0.bias")
    X4 = layer(mm(X3, tr(W["mid2.0.0"])), "mid2.0.0.bias")
    XC = layer(mm(X4, tr(W["color_linear.0"][..., :H])) + mm(emb2, tr(W["color_linear.0"][..., H:])),
               "color_linear.0.bias")
    raw_a = (mm(X4, w_a[..., None])[..., 0] + p["out_alpha.bias"]) * 10.0
    raw_c = mm(XC, tr(W_oc)) + p["out_color.bias"][:, None, :]
    return X1, X2, X3, X4, XC, raw_a, raw_c


def _params64(params, dev):
    return {k: v.to(dtype=torch.float64, device=dev) for k, v in params.items()}


def fused_forward(params: Dict[str, torch.Tensor], scale, points: torch.Tensor,
                  emb: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, rounding: Rounding = ROUND_ALL):
    """What ``eval_points`` returns at hidden 32: raw alpha x10 [B,N] and sigmoid colour [B,N,3], in fp64.
    points [B,N,3]; emb: optional (E1, E2) in the reference column order."""
    dev = points.device
    p = _params64(params, dev)
    if emb is None:
        emb = embedding(points[:, :, None], p[PE_KEY], scale, rounding)
    W, w_a, W_oc = _weights(p, rounding)
    *_, raw_a, raw_c = _mlp(p, W, w_a, W_oc, emb[0].to(p[PE_KEY]), emb[1].to(p[PE_KEY]), rounding)
    return raw_a, torch.sigmoid(raw_c)


def fused_step(params: Dict[str, torch.Tensor], scale, batch: Dict[str, torch.Tensor],
               counts: Optional[torch.Tensor] = None, signs: Optional[torch.Tensor] = None,
               emb: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, var: Optional[torch.Tensor] = None,
               rounding: Rounding = ROUND_ALL, ls: float = LS, colour_scaling: float = 5.0, opacity_scaling: float = 10.0, aux: Optional[dict] = None):
    """One fused hidden-32 step of a stack of objects (forward, render, losses, gradients; no AdamW).

    params: stacked ``[B, *shape]`` fp32 master weights keyed by ``vmap_oracle.ALL_KEYS``; scale: scalar or [B];
    batch: the six step inputs; counts: [B,4] mask counts (default: from this batch); signs: [B,R,5] residual signs;
    emb: (E1 [B,R*S,87], E2 [B,R*S,42]) to use as the embedding (the kernel's own, see ``tests/test_fused_faithful_gpu``);
    var: [B,R] ray variances for the depth-loss weight 1 / (sqrt(var) + 1e-4) (e.g. the kernel's: the fp32 sum
    cancels on rays whose weight sits on one sample, and the weight amplifies that); ls: the loss scale; aux: a dict
    that receives ``dh`` (``ls * dh`` before its fp16 pack, [B,P,4]), ``dproj`` ([B,P,21], before its fp16 pack) and
    ``dt`` (each point's dL/dt = ``INV_LS (dE1_xyz + dproj @ dirs)`` [B,P,3] from that unrounded dproj, as the joint
    step's ``pe_backward`` forms it).
    Returns ``(render, loss_terms, grads)`` as ``oracle.lw_oracle.lw_step`` does; all fp64."""
    dev = batch["pcs"].device
    f64 = dict(dtype=torch.float64, device=dev)
    rnd = rounding
    inv_ls = 1.0 / ls
    p = _params64(params, dev)
    pcs = batch["pcs"]
    B, R, S, _ = pcs.shape
    P = R * S
    mm, tr = torch.matmul, (lambda x: x.transpose(1, 2))

    # ---- E0: embedding ----
    t, proj = projections(pcs, p[PE_KEY], scale, rnd.proj32)
    if emb is None:
        band = sin_bands(proj)
        emb1 = _half(torch.cat([t, band[..., :4 * N_DIRS]], -1), rnd.emb)
        emb2 = _half(band[..., 4 * N_DIRS:], rnd.emb)
    else:
        emb1, emb2 = emb[0].to(**f64), emb[1].to(**f64)

    # ---- forward stages 1..7 ----
    W, w_a, W_oc = _weights(p, rnd)
    H = W["mid1.0.0"].shape[-1]
    X1, X2, X3, X4, XC, raw_a, raw_c = _mlp(p, W, w_a, W_oc, emb1, emb2, rnd)

    # ---- heads + volume render + losses + ray gradients ----
    oc = torch.sigmoid(raw_a).reshape(B, R, S)
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
    on = (cnt[:, :3] != 0).all(0).double()                                             # any-empty early-out
    inv = 1.0 / (cnt[:, :3].float() + 1e-10).double()
    m_o = (sem != 0).double()
    m_s = (sem != 2).double()
    m_d = mask.bool().double() * m_o
    info = 1.0 / (torch.sqrt(V if var is None else var.to(**f64)) + 1e-4)
    e_d = D - batch["gt_depth"].to(**f64)
    e_c = C - batch["gt_colour"].to(**f64)
    e_o = O - m_o
    l_d = on[0] * (e_d.abs() * m_d * info).sum(1) * inv[:, 0]
    l_c = on[1] * (e_c.abs().sum(-1) * m_o).sum(1) * inv[:, 1]
    l_o = on[2] * (e_o.abs() * m_s).sum(1) * inv[:, 2]
    loss_terms = torch.stack([l_d, l_c, l_o, l_d + colour_scaling * l_c + opacity_scaling * l_o], 1)
    sg = torch.cat([e_d[..., None], e_c, e_o[..., None]], -1).sign() if signs is None else signs.to(**f64)

    # the loss scale enters at the loss gradient
    gD = ls * on[0] * sg[..., 0] * m_d * info * inv[:, :1]                             # [B,R]
    gC = (ls * on[1] * colour_scaling * m_o * inv[:, 1:2])[..., None] * sg[..., 1:4]   # [B,R,3]
    gO = ls * on[2] * opacity_scaling * sg[..., 4] * m_s * inv[:, 2:3]
    Gs = gD[..., None] * z + (gC[..., None, :] * col).sum(-1) + gO[..., None]
    gw = Gs * w
    suffix = gw.flip(-1).cumsum(-1).flip(-1) - gw
    docc = Gs * T - suffix / om
    dh_a = (10.0 * docc * oc * (1.0 - oc)).reshape(B, P)
    dh_c = (gC[..., None, :] * w[..., None] * col * (1.0 - col)).reshape(B, P, 3)
    dh = torch.cat([dh_a[..., None], dh_c], -1)                                        # ls * dh, fp32 in the kernel
    if aux is not None:
        aux["dh"] = dh
    dh16 = _half(dh, rnd.dh, rnd.dh_lim)
    feed = dh16 if rnd.dh_feeds else dh                                                # into dYc, dY4 and the head biases

    g = {}
    g["out_alpha.weight"] = inv_ls * mm(tr(dh16[..., :1]), X4)
    g["out_alpha.bias"] = inv_ls * feed[..., 0].sum(1, keepdim=True)
    g["out_color.weight"] = inv_ls * mm(tr(dh16[..., 1:]), XC)
    g["out_color.bias"] = inv_ls * feed[..., 1:].sum(1)

    # ---- backward stages ----
    def gate(acc, x_prev, on_, lim=HALF_MAX):
        return _half(acc, on_, lim) * (x_prev > 0)

    def wgrad(dY, X, key):
        g[key + ".weight"] = inv_ls * mm(tr(dY), X)
        g[key + ".bias"] = inv_ls * dY.sum(1)

    W_cl, W_cat = W["color_linear.0"], W["cat_layer.0"]
    dYc = gate(mm(feed[..., 1:], W_oc), XC, rnd.dyc, rnd.dh_lim)
    dY4 = gate(mm(dYc, W_cl[..., :H]) + feed[..., :1] * w_a[:, None, :], X4, rnd.dgrad)
    wgrad(dYc, torch.cat([X4, emb2], -1), "color_linear.0")
    dE2 = mm(dYc, W_cl[..., H:])
    dY3 = gate(mm(dY4, W["mid2.0.0"]), X3, rnd.dgrad)
    wgrad(dY4, X3, "mid2.0.0")
    dY2 = gate(mm(dY3, W_cat[..., :H]), X2, rnd.dgrad)
    wgrad(dY3, torch.cat([X2, emb1], -1), "cat_layer.0")
    dY1 = gate(mm(dY2, W["mid1.0.0"]), X1, rnd.dgrad)
    wgrad(dY2, X1, "mid1.0.0")
    wgrad(dY1, emb1, "in_layer.0")
    dE1 = mm(dY3, W_cat[..., H:]) + mm(dY1, W["in_layer.0"])

    # ---- PE backward and dB ----
    dband = torch.cat([dE1[..., 3:], dE2], -1)                                         # [B,P,126] frequency-major
    cb = cos_bands(proj, rnd.cos32)
    pi = PI_F if rnd.cos32 else math.pi
    dproj = sum(dband[..., k * N_DIRS:(k + 1) * N_DIRS] * (2.0 ** k) * cb[k] for k in range(N_BANDS)) * pi
    if aux is not None:                                                                # pe_backward: from fp32 dproj
        aux["dproj"] = dproj
        aux["dt"] = inv_ls * (dE1[..., :3] + mm(dproj, p[PE_KEY]))
    dproj = _half(dproj, rnd.dproj)
    tt = emb1[..., :3] if (rnd.t16 and emb is not None) else _half(t, rnd.t16)
    g[PE_KEY] = inv_ls * mm(tr(dproj), tt)

    render = (D, V, C, O)
    return render, loss_terms, {k: g[k].reshape(params[k].shape) for k in ALL_KEYS}
