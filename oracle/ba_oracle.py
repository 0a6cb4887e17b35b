"""CPU restatement (torch fp64) of the bundle-adjustment rule of ``vmap_b200/csrc/k_ba.cuh`` (K11).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

It builds on ``track_oracle`` (K10's restatement) and generalises it from one pose to a pose per ray: every group's
batch carries ``frames`` [B,R], the row of a pose table ``poses`` [F,4,4] each ray is seen from (-1: the ray contributes
nothing).  The loss is K10's, unchanged; the gradient is the left-perturbation tangent ``(phi_f, rho_f)`` of every
frame, taken by fp64 autograd at zero tangents.  The update is one Adam over the stacked tangents of a window of frames,
with a held frame that never moves.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import torch

from . import track_oracle as to
from . import vmap_oracle as vo


def _split(g):
    params, scale, b = to._f64(g)
    frames = torch.as_tensor(g["batch"]["frames"], dtype=torch.int64)
    return params, scale, b, frames


def _points(q, frames, R, t):
    """p = R_f q + t_f per ray ([B,R,S,3]); rays with frame -1 get frame 0's pose (their loss is masked)."""
    f = frames.clamp(min=0)
    Rr, tr = R[f], t[f]                                            # [B,R,3,3], [B,R,3]
    return torch.einsum("brij,brsj->brsi", Rr, q) + tr[:, :, None, :]


def _loss_terms(alpha, colour, b, ok, var=None):
    """track_oracle.loss_terms with K11's guard: a ray with no frame (``ok`` False) leaves every term, while the
    per-object counts stay those of the whole slice (the kernel counts before it looks a ray's frame up)."""
    sem, md = b["sem"], b["mask_depth"]
    m_obj = (sem != 0) & ok
    m_sem = (sem != 2) & ok
    depth, var_here, col, opa = vo.render_outputs(alpha, colour, b["z"])
    var = var_here.detach() if var is None else var
    m_d = md.bool() & m_obj
    cnt_d, cnt_o, cnt_s = (b["mask_depth"].bool() & (b["sem_raw"] != 0)), b["sem_raw"] != 0, b["sem_raw"] != 2
    l_d = _mean(((depth - b["gt_depth"]).abs() * m_d) / (torch.sqrt(var) + 1e-4), cnt_d)
    l_c = _mean((col - b["gt_colour"]).abs().sum(-1) * m_obj, cnt_o)
    l_o = _mean((opa - m_obj.to(opa.dtype)).abs() * m_sem, cnt_s)
    return torch.stack([l_d, l_c, l_o], dim=1)


def _mean(x, mask):
    """Per object and per term: sum / (count + 1e-10), 0 where the term's own count is 0."""
    cnt = mask.sum(-1)
    out = x.sum(-1) / (cnt + 1e-10)
    return torch.where(cnt > 0, out, torch.zeros_like(out))


def _prep(b, frames):
    ok = frames >= 0
    out = dict(b)
    out["sem_raw"] = b["sem"]
    return out, ok


def evaluate(groups: Sequence[Dict], poses, cs: float = 5.0, os_: float = 10.0):
    """Loss, per-frame tangent gradients and per-point magnitudes at the pose table ``poses`` [F,4,4].

    Returns ``(loss, grad [F,6] (phi, rho), abs_sum [F,6], terms)``; ``abs_sum[f]`` is the sum over frame f's points of
    |per-point contribution|, the scale of the cancellation in its sum."""
    P = torch.as_tensor(np.asarray(poses, np.float64))
    F = P.shape[0]
    R0, t0 = P[:, :3, :3], P[:, :3, 3]
    xi = torch.zeros(F, 6, dtype=torch.float64, requires_grad=True)
    R = torch.stack([to.exp_so3(xi[f, :3]) @ R0[f] for f in range(F)])
    t = t0 + xi[:, 3:]
    total = torch.zeros((), dtype=torch.float64)
    pts, terms = [], []
    for g in groups:
        params, scale, b, frames = _split(g)
        b, ok = _prep(b, frames)
        p = _points(b["pcs"], frames, R, t)
        p.retain_grad()
        alpha, colour = vo.forward(params, scale, p)
        lt = _loss_terms(alpha, colour, b, ok)
        tot = lt[:, 0] + cs * lt[:, 1] + os_ * lt[:, 2]
        total = total + tot.sum()
        terms.append(torch.cat([lt, tot[:, None]], 1).detach())
        pts.append((p, b["pcs"], frames))
    total.backward()
    abs_sum = torch.zeros(F, 6, dtype=torch.float64)
    for p, q, frames in pts:
        f = frames.clamp(min=0)
        rq = torch.einsum("brij,brsj->brsi", R0[f], q)
        c = torch.cat([torch.cross(rq, p.grad, dim=-1), p.grad], -1).abs().sum(2)      # [B,R,6]
        c = c * (frames >= 0)[..., None]
        abs_sum.index_add_(0, f.reshape(-1), c.reshape(-1, 6))
    return float(total.detach()), xi.grad.detach().numpy().copy(), abs_sum.numpy(), terms


def loss_at(groups, poses, cs: float = 5.0, os_: float = 10.0, var_poses=None) -> float:
    """The loss at ``poses``; with ``var_poses`` the depth weights are the variances rendered there (held fixed)."""
    P = torch.as_tensor(np.asarray(poses, np.float64))
    Pv = None if var_poses is None else torch.as_tensor(np.asarray(var_poses, np.float64))
    total = 0.0
    with torch.no_grad():
        for g in groups:
            params, scale, b, frames = _split(g)
            b, ok = _prep(b, frames)
            alpha, colour = vo.forward(params, scale, _points(b["pcs"], frames, P[:, :3, :3], P[:, :3, 3]))
            var = None
            if Pv is not None:
                av, cv = vo.forward(params, scale, _points(b["pcs"], frames, Pv[:, :3, :3], Pv[:, :3, 3]))
                var = vo.render_outputs(av, cv, b["z"])[1]
            lt = _loss_terms(alpha, colour, b, ok, var)
            total += float((lt[:, 0] + cs * lt[:, 1] + os_ * lt[:, 2]).sum())
    return total


def window_update(poses, window: Sequence[int], grads, m, v, it: int, lr_rot: float, lr_trans: float,
                  hold: int = 0, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8):
    """One Adam step over the stacked tangents of the window frames (``grads`` [F,6] indexed by frame; ``m``, ``v``
    [len(window),6], zero before it = 1), then each frame's retraction.  ``hold`` never moves."""
    P = np.array(poses, np.float64, copy=True)
    m = np.zeros((len(window), 6)) if it == 1 else np.array(m, np.float64, copy=True)
    v = np.zeros((len(window), 6)) if it == 1 else np.array(v, np.float64, copy=True)
    for w, f in enumerate(window):
        if f == hold:
            continue
        P[f], m[w], v[w] = to.adam_update(P[f], grads[f], m[w] if it > 1 else None, v[w] if it > 1 else None, it,
                                          lr_rot, lr_trans, b1, b2, eps)
    return P, m, v


def slice_groups(groups: Sequence[Dict], it: int, n_pix: Sequence[int]) -> List[Dict]:
    """Iteration ``it`` uses rays [it * n_pix, (it + 1) * n_pix) of every group (frames included)."""
    return to.slice_groups(groups, it, n_pix)


def bundle_adjust(groups, poses, window: Sequence[int], n_iter: int, n_pix: Sequence[int], lr_rot: float,
                  lr_trans: float, hold: int = 0):
    """The whole pass; returns (poses [n_iter+1,F,4,4], losses [n_iter], grads [n_iter,F,6])."""
    P = np.asarray(poses, np.float64)
    m = v = None
    hist, losses, grads = [P], [], []
    for it in range(n_iter):
        loss, g, _, _ = evaluate(slice_groups(groups, it, n_pix), P)
        losses.append(loss)
        grads.append(g)
        gw = np.stack([g[f] for f in window if f != hold]) if any(f != hold for f in window) else np.zeros((0, 6))
        if np.isfinite(loss) and np.all(np.isfinite(gw)):
            P, m, v = window_update(P, window, g, m, v, it + 1, lr_rot, lr_trans, hold)
        elif it == 0:
            m = v = np.zeros((len(window), 6))
        hist.append(P)
    return np.stack(hist), np.array(losses), np.stack(grads)
