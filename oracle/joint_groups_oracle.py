"""CPU restatement (torch fp64) of the joint map-and-pose iterations over several groups that share one pose table:
the vMAP objects' ``vmb_joint_step_fused`` (csrc/k_step_fused.cuh, csrc/k_track_lw.cuh) and the background model's
``vmb_joint_step_lw``, into one ``vmb_ba_update``.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

Each group is ``joint_oracle.joint``'s one group (camera-frame ``pcs`` and the ``frames`` each ray is seen from); the
pose gradient of an iteration is taken over all groups at once, as the update sums both groups' rows.
"""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np
import torch

from . import ba_oracle as bo
from . import vmap_oracle as vo
from .joint_oracle import world_batch


def joint_groups(groups: Sequence[Dict], poses, window: Sequence[int], n_iter: int, n_pix: Sequence[int], lr: float,
                 weight_decay: float, lr_rot: float, lr_trans: float, hold: int = 0):
    """``joint`` over several groups that share one pose table (vMAP: the hidden-32 objects and the background model,
    ``vmb_joint_step_fused`` + ``vmb_joint_step_lw`` into one ``vmb_ba_update``).  ``groups``: dicts of ``params``,
    ``scale`` and ``batch`` (with ``frames``); group k's iteration ``it`` uses rays [it * n_pix[k], (it + 1) * n_pix[k]).
    Per iteration: the pose gradient of every frame over all groups (``ba_oracle.evaluate`` on the list), each group's
    mapping step with AdamW on its world points, one Adam + Exp over the window.  Returns dict(params (a list, one per
    group, after the last iteration), poses [n_iter+1,F,4,4], losses [n_iter] (the sum of the groups' mapping losses),
    pose_grads [n_iter,F,6])."""
    enss = [vo.OracleEnsemble({k: torch.as_tensor(v, dtype=torch.float64) for k, v in g["params"].items()},
                              torch.as_tensor(g["scale"], dtype=torch.float64), lr=lr, weight_decay=weight_decay)
            for g in groups]
    P = np.asarray(poses, np.float64)
    m = v = None
    hist, losses, grads = [P], [], []
    for it in range(n_iter):
        sl = bo.slice_groups(list(groups), it, list(n_pix))
        cur = [{"params": {k: t.detach() for k, t in e.params.items()}, "scale": e.scale, "batch": s["batch"]}
               for e, s in zip(enss, sl)]
        _, g, _, _ = bo.evaluate(cur, P)
        losses.append(sum(float(e.step(world_batch(s["batch"], P))) for e, s in zip(enss, sl)))
        grads.append(g)
        gw = np.stack([g[f] for f in window if f != hold]) if any(f != hold for f in window) else np.zeros((0, 6))
        if np.all(np.isfinite(gw)):
            P, m, v = bo.window_update(P, window, g, m, v, it + 1, lr_rot, lr_trans, hold)
        elif it == 0:
            m = v = np.zeros((len(window), 6))
        hist.append(P)
    return {"params": [{k: t.detach() for k, t in e.params.items()} for e in enss], "poses": np.stack(hist),
            "losses": np.array(losses), "pose_grads": np.stack(grads)}
