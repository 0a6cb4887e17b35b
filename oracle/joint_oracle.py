"""CPU restatement (torch fp64) of the joint map-and-pose iterations of ``vmb_joint_step_lw`` (csrc/k_track_lw.cuh).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

One group of objects whose batch holds camera-frame points ``pcs`` [B,N,S,3] and ``frames`` [B,N] (the row of the pose
table each ray is seen from).  Iteration ``it`` uses rays [it * n_pix, (it + 1) * n_pix) and, in this order:

    the pose gradient of every frame at the current weights (``ba_oracle.evaluate``),
    the mapping step on the world points p = R_f q + t_f and AdamW on the weights (``vmap_oracle.OracleEnsemble.step``),
    one Adam + Exp over the window of poses (``ba_oracle.window_update``); ``hold`` never moves.

Both gradients are taken at the weights and poses the iteration starts from, as the kernel takes them from one
forward and backward.  The pose moments start at zero (the kernel's restart with every mapping frame).
"""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np
import torch

from . import ba_oracle as bo
from . import vmap_oracle as vo


def world_batch(batch: Dict[str, torch.Tensor], poses) -> Dict[str, torch.Tensor]:
    """``batch`` with ``pcs`` moved to the world by each ray's frame (fp64; frame -1 takes frame 0's pose)."""
    P = torch.as_tensor(np.asarray(poses, np.float64))
    out = {k: v for k, v in batch.items() if k != "frames"}
    out["pcs"] = bo._points(torch.as_tensor(batch["pcs"], dtype=torch.float64),
                            torch.as_tensor(batch["frames"], dtype=torch.int64), P[:, :3, :3], P[:, :3, 3])
    for k in ("z", "gt_depth", "gt_colour"):
        out[k] = torch.as_tensor(batch[k], dtype=torch.float64)
    return out


def joint(params: Dict[str, torch.Tensor], scale, batch: Dict[str, torch.Tensor], poses, window: Sequence[int],
          n_iter: int, n_pix: int, lr: float, weight_decay: float, lr_rot: float, lr_trans: float, hold: int = 0):
    """n_iter joint iterations.  Returns dict(params (after the last iteration, fp64), poses [n_iter+1,F,4,4],
    losses [n_iter] (the mapping loss of each iteration), pose_grads [n_iter,F,6])."""
    p64 = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in params.items()}
    ens = vo.OracleEnsemble(p64, torch.as_tensor(scale, dtype=torch.float64), lr=lr, weight_decay=weight_decay)
    P = np.asarray(poses, np.float64)
    m = v = None
    hist, losses, grads = [P], [], []
    for it in range(n_iter):
        sl = bo.slice_groups([{"params": params, "scale": scale, "batch": batch}], it, [n_pix])[0]
        cur = {k: t.detach() for k, t in ens.params.items()}
        _, g, _, _ = bo.evaluate([{"params": cur, "scale": ens.scale, "batch": sl["batch"]}], P)
        losses.append(float(ens.step(world_batch(sl["batch"], P))))
        grads.append(g)
        gw = np.stack([g[f] for f in window if f != hold]) if any(f != hold for f in window) else np.zeros((0, 6))
        if np.all(np.isfinite(gw)):
            P, m, v = bo.window_update(P, window, g, m, v, it + 1, lr_rot, lr_trans, hold)
        elif it == 0:
            m = v = np.zeros((len(window), 6))
        hist.append(P)
    return {"params": {k: t.detach() for k, t in ens.params.items()}, "poses": np.stack(hist),
            "losses": np.array(losses), "pose_grads": np.stack(grads)}
