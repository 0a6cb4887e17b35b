"""Generate tests/golden/ref_track.npz from the UNMODIFIED reference (needs a reference checkout, see
oracle/_refload.py).

Run:  python -m oracle.make_track_golden        (no GPU)

The tracking loss of K10 (csrc/k_track.cuh) is the training loss of every tracked object at world points
p = R q + t.  Here it is evaluated in fp64 by the reference's own ``embedding.UniDirsEmbed``, ``model.OccupancyMap``
and ``loss.step_batch_loss``, driven as train.py:293-303 drives them (functorch ``combine_state_for_ensemble`` +
``vmap``), and differentiated by autograd with respect to a zero left-perturbation tangent (phi, rho):
R <- Exp(phi) R, t <- t + rho.  Every mask of both cases is non-empty, so the reference's whole-batch empty-mask rule
and the package's per-object rule agree.  Cases: three hidden-32 objects (S = 10) and one hidden-128 background
(S = 14).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import _refload  # noqa: E402
from oracle import track_oracle as to  # noqa: E402
from oracle import vmap_oracle as vo  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CASES = (("obj", 3, 32, 10, 1, 2.0, 40), ("bg", 1, 128, 14, 5, 5.0, 60))


def _pose(seed):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    w *= np.radians(15.0) / np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w)
    T[:3, 3] = rng.uniform(-0.3, 0.3, 3)
    return T


def reference_track_case(tag, n_obj, hidden, S, n1, scale, n_rays, seed, out):
    model, embedding, loss = _refload.load("model", "embedding", "loss")
    from functorch import combine_state_for_ensemble, vmap

    torch.manual_seed(seed)
    e1, e2 = vo.emb_sizes(5)
    fcs, pes = [], []
    for _ in range(n_obj):                                          # trainer.py:27-33
        fc = model.OccupancyMap(e1, e2, hidden_size=hidden)
        fc.apply(model.init_weights)
        fcs.append(fc.double())
        pes.append(embedding.UniDirsEmbed(max_deg=5, scale=scale).double())
    batch = vo.synthetic_batch(n_obj, n_rays, S, seed=seed + 100, n_cam2surf=n1, dtype=torch.float64)
    assert bool((batch["sem"] != 0).any(1).all() and (batch["sem"] != 2).any(1).all())      # every mask non-empty
    assert bool(((batch["sem"] != 0) & batch["mask_depth"]).any(1).all())
    fc_model, fc_param, fc_buffer = combine_state_for_ensemble(fcs)
    pe_model, pe_param, pe_buffer = combine_state_for_ensemble(pes)
    T = torch.from_numpy(_pose(seed))
    xi = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    R = to.exp_so3(xi[:3]) @ T[:3, :3]
    t = T[:3, 3] + xi[3:]
    pcs = batch["pcs"] @ R.transpose(0, 1) + t                      # p = R q + t, q = the identity-pose samples
    emb = vmap(pe_model)(pe_param, pe_buffer, pcs)                  # train.py:293
    alpha, col = vmap(fc_model)(fc_param, fc_buffer, emb)           # train.py:294
    l, _ = loss.step_batch_loss(alpha, col, batch["gt_depth"], batch["gt_colour"], batch["sem"],
                                batch["mask_depth"], batch["z"])    # train.py:303
    l.backward()
    assert emb.dtype == torch.float64 and alpha.dtype == torch.float64
    fc_names = [n for n, _ in fcs[0].named_parameters()]
    assert tuple(fc_names) == vo.FC_KEYS, fc_names
    for n, p in zip(fc_names, fc_param):
        out[f"{tag}_p_{n}"] = p.detach().numpy().copy()
    out[f"{tag}_p_{vo.PE_KEY}"] = pe_param[0].detach().numpy().copy()
    for k, v in batch.items():
        out[f"{tag}_in_{k}"] = v.numpy().copy()
    out[f"{tag}_scale"] = np.float64(scale)
    out[f"{tag}_pose"] = T.numpy().copy()
    out[f"{tag}_loss"] = np.float64(l.detach())
    out[f"{tag}_grad"] = xi.grad.numpy().copy()
    print(tag, "loss", float(l), "grad", xi.grad.numpy())


def main():
    out = {}
    for i, (tag, n_obj, hidden, S, n1, scale, n_rays) in enumerate(CASES):
        reference_track_case(tag, n_obj, hidden, S, n1, scale, n_rays, 900 + i, out)
    np.savez_compressed(os.path.join(OUT, "ref_track.npz"), **out)


if __name__ == "__main__":
    main()
