"""CPU restatement (torch fp64) of the tracking rule of ``vmap_b200/csrc/k_track.cuh`` (K10).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

A *group* is one ensemble's share of a frame: ``{"params": stacked dict [B,...], "scale": [B], "batch": {...}}`` with
``batch["pcs"]`` the camera-frame points ``q`` [B,R,S,3] of the identity-pose samples and the usual z / gt_depth /
gt_colour / sem / mask_depth.  The pose is camera-to-world ``T_wc`` [4,4]; the world point is ``p = R q + t``.
The loss is the training loss of every object (vmap_oracle.batch_loss_terms) except for the empty-mask rule, which is
per object and per term here.  The gradient is the left-perturbation tangent ``(phi, rho)``:
``R <- Exp(phi) R, t <- t + rho``, taken by fp64 autograd at a zero tangent.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import vmap_oracle as vo

EXP_SMALL = 1e-12


def hat(w: torch.Tensor) -> torch.Tensor:
    z = torch.zeros((), dtype=w.dtype)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]),
                        torch.stack([-w[1], w[0], z])])


def exp_so3(w: torch.Tensor) -> torch.Tensor:
    """Rodrigues in fp64; I + [w]x below |w| = 1e-12 (differentiable at 0)."""
    th = torch.linalg.norm(w)
    K = hat(w)
    eye = torch.eye(3, dtype=w.dtype)
    if float(th.detach()) < EXP_SMALL:
        return eye + K
    return eye + torch.sin(th) / th * K + (1.0 - torch.cos(th)) / (th * th) * (K @ K)


def exp_so3_np(w) -> np.ndarray:
    return exp_so3(torch.as_tensor(np.asarray(w, np.float64))).numpy()


def _masked_mean_per_object(loss_mat, mask, info=None):
    """Per object and per term: a term whose own mask count is 0 contributes 0 for that object only."""
    cnt = mask.sum(-1)
    if info is not None:
        loss_mat = loss_mat * info
    out = loss_mat.sum(-1) / (cnt + 1e-10)
    return torch.where(cnt > 0, out, torch.zeros_like(out))


def loss_terms(alpha, colour, batch, var=None) -> torch.Tensor:
    """[B,3] (L_depth, L_colour, L_opacity) with the per-object empty-mask rule (loss.py:5-56 otherwise).
    ``var``: the (detached) rendered variance to weight the depth term with, instead of this render's."""
    sem, md = batch["sem"], batch["mask_depth"]
    m_obj = sem != 0
    m_sem = sem != 2
    depth, var_here, col, opa = vo.render_outputs(alpha, colour, batch["z"])
    var = var_here.detach() if var is None else var
    m_d = md.bool() & m_obj
    l_d = _masked_mean_per_object((depth - batch["gt_depth"]).abs() * m_d, m_d, info=1.0 / (torch.sqrt(var) + 1e-4))
    l_c = _masked_mean_per_object((col - batch["gt_colour"]).abs().sum(-1) * m_obj, m_obj)
    l_o = _masked_mean_per_object((opa - m_obj.to(opa.dtype)).abs() * m_sem, m_sem)
    return torch.stack([l_d, l_c, l_o], dim=1)


def _f64(group):
    p = {k: v.detach().to(torch.float64) for k, v in group["params"].items()}
    b = {k: (v.to(torch.float64) if v.is_floating_point() else v) for k, v in group["batch"].items()}
    return p, torch.as_tensor(group["scale"], dtype=torch.float64).reshape(-1), b


def _world(q, R, t):
    return q @ R.transpose(0, 1) + t


def evaluate(groups: Sequence[Dict], T_wc, cs: float = 5.0, os_: float = 10.0):
    """Loss, tangent gradient and per-point magnitudes at pose ``T_wc``.

    Returns ``(loss, grad [6] (phi, rho), abs_sum [6], terms)``: ``abs_sum`` is sum over points of |per-point
    contribution| (the scale of the cancellation in the sum), ``terms`` a list of [B,4] per-object loss terms."""
    T = torch.as_tensor(np.asarray(T_wc, np.float64))
    R0, t0 = T[:3, :3], T[:3, 3]
    xi = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    R = exp_so3(xi[:3]) @ R0
    t = t0 + xi[3:]
    total = torch.zeros((), dtype=torch.float64)
    pts, terms = [], []
    for g in groups:
        params, scale, b = _f64(g)
        p = _world(b["pcs"], R, t)
        p.retain_grad()
        alpha, colour = vo.forward(params, scale, p)
        lt = loss_terms(alpha, colour, b)
        tot = lt[:, 0] + cs * lt[:, 1] + os_ * lt[:, 2]
        total = total + tot.sum()
        terms.append(torch.cat([lt, tot[:, None]], 1).detach())
        pts.append((p, b["pcs"]))
    total.backward()
    abs_sum = torch.zeros(6, dtype=torch.float64)
    for p, q in pts:
        gp = p.grad
        rq = q @ R0.transpose(0, 1)
        c = torch.cat([torch.cross(rq, gp, dim=-1), gp], -1).reshape(-1, 6)
        abs_sum += c.abs().sum(0)
    return float(total.detach()), xi.grad.detach().numpy().copy(), abs_sum.numpy(), terms


def loss_at(groups, T_wc, cs: float = 5.0, os_: float = 10.0, var_pose=None) -> float:
    """The loss at ``T_wc``; with ``var_pose`` the depth term's variance weights are those rendered at ``var_pose``
    (held constant, as the detached variance is for the gradient: what central differences must hold fixed)."""
    T = torch.as_tensor(np.asarray(T_wc, np.float64))
    Tv = None if var_pose is None else torch.as_tensor(np.asarray(var_pose, np.float64))
    total = 0.0
    with torch.no_grad():
        for g in groups:
            params, scale, b = _f64(g)
            alpha, colour = vo.forward(params, scale, _world(b["pcs"], T[:3, :3], T[:3, 3]))
            var = None
            if Tv is not None:
                av, cv = vo.forward(params, scale, _world(b["pcs"], Tv[:3, :3], Tv[:3, 3]))
                var = vo.render_outputs(av, cv, b["z"])[1]
            lt = loss_terms(alpha, colour, b, var)
            total += float((lt[:, 0] + cs * lt[:, 1] + os_ * lt[:, 2]).sum())
    return total


def retract(T_wc, xi) -> np.ndarray:
    """T <- (Exp(phi) R, t + rho)."""
    T = np.array(T_wc, np.float64, copy=True)
    T[:3, :3] = exp_so3_np(xi[:3]) @ T[:3, :3]
    T[:3, 3] = T[:3, 3] + np.asarray(xi[3:], np.float64)
    return T


def adam_update(T_wc, g, m, v, it: int, lr_rot: float, lr_trans: float, b1: float = 0.9, b2: float = 0.999,
                eps: float = 1e-8) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """One Adam step on the tangent (no weight decay; m = v = 0 before it = 1), then the retraction."""
    g = np.asarray(g, np.float64)
    m = (np.zeros(6) if it == 1 else b1 * np.asarray(m, np.float64)) + (1.0 - b1) * g
    v = (np.zeros(6) if it == 1 else b2 * np.asarray(v, np.float64)) + (1.0 - b2) * g * g
    bc1, bc2 = 1.0 - b1 ** it, 1.0 - b2 ** it
    lr = np.array([lr_rot] * 3 + [lr_trans] * 3)
    d = -lr * (m / bc1) / (np.sqrt(v / bc2) + eps)
    return retract(T_wc, d), m, v


def slice_groups(groups: Sequence[Dict], it: int, n_pix: Sequence[int]) -> List[Dict]:
    """Iteration ``it`` uses draw ``it``: rays [it * n_pix, (it + 1) * n_pix) of every group."""
    out = []
    for g, n in zip(groups, n_pix):
        out.append({"params": g["params"], "scale": g["scale"],
                    "batch": {k: v[:, it * n:(it + 1) * n] for k, v in g["batch"].items()}})
    return out


def track(groups, T_init, n_iter: int, n_pix: Sequence[int], lr_rot: float, lr_trans: float):
    """The whole loop; returns (poses [n_iter+1,4,4], losses [n_iter], grads [n_iter,6])."""
    T = np.asarray(T_init, np.float64)
    m = v = np.zeros(6)
    poses, losses, grads = [T], [], []
    for it in range(n_iter):
        loss, g, _, _ = evaluate(slice_groups(groups, it, n_pix), T)
        losses.append(loss)
        grads.append(g)
        if np.isfinite(loss) and np.all(np.isfinite(g)):
            T, m, v = adam_update(T, g, m, v, it + 1, lr_rot, lr_trans)
        poses.append(T)
    return np.stack(poses), np.array(losses), np.stack(grads)


def rot_err_deg(Ra, Rb) -> float:
    c = (np.trace(np.asarray(Ra).T @ np.asarray(Rb)) - 1.0) / 2.0
    return math.degrees(math.acos(max(-1.0, min(1.0, c))))
