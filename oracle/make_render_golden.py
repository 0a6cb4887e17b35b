"""Generate tests/golden/ref_render.npz: the reference's own arithmetic on the renderer's samples.  The geometry
(hits, coarse samples, fine positions) is the oracle's (oracle/render_oracle.py, the rule of k_render.cuh); the
networks are the reference's ``embedding.UniDirsEmbed`` + ``model.OccupancyMap`` with the golden scene's parameters,
and each ray's merged sequence is composited with ``render_rays.occupancy_activation`` /
``occupancy_to_termination(is_batch=False)`` / ``render``.  The surface is the first sample whose running sum of the
reference's termination weights reaches 0.5; it drives the fine pass.  Needs a reference checkout (see
oracle/_refload.py); no GPU.  Touches no other golden.

Run:  python -m oracle.make_render_golden
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import _refload  # noqa: E402
from oracle import render_oracle as ro  # noqa: E402
from oracle import vmap_oracle as vo  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_render.npz")


def reference_nets(nets):
    model, embedding = _refload.load("model", "embedding")
    e1, e2 = vo.emb_sizes(5)
    out = []
    for p, scale in nets:
        hidden = p["mid1.0.0.weight"].shape[1]
        fc = model.OccupancyMap(e1, e2, hidden_size=hidden)
        pe = embedding.UniDirsEmbed(max_deg=5, scale=scale)
        with torch.no_grad():
            for k, v in fc.named_parameters():
                v.copy_(p[k][0])
            pe.B_layer.weight.copy_(p[vo.PE_KEY][0])

        def f(pts, fc=fc, pe=pe):
            with torch.no_grad():
                a, c = fc(pe(torch.from_numpy(np.ascontiguousarray(pts, np.float32))))
            return a.reshape(-1).numpy(), c.reshape(-1, 3).numpy()
        out.append(f)
    return out


def reference_composite(n, src, ids, passes, rr):
    per_ray = [[] for _ in range(n)]
    for p, (smp, alpha, col) in enumerate(passes):
        for j, (r, i, k) in enumerate(smp["meta"]):
            per_ray[r].append((float(smp["z"][j]), int(src[r, i]), p, int(k), j))
    out = {"depth": np.zeros(n, np.float32), "colour": np.zeros((n, 3), np.float32),
           "opacity": np.zeros(n, np.float32), "instance": np.full(n, -1, np.int32),
           "zstar": np.full(n, -1.0, np.float32), "acc_at_surf": np.full(n, np.nan)}
    for r in range(n):
        seq = sorted(per_ray[r])
        if not seq:
            continue
        z = torch.tensor([x[0] for x in seq], dtype=torch.float32)[None]
        a = torch.from_numpy(np.array([passes[x[2]][1][x[4]] for x in seq], np.float32))[None]
        c = torch.from_numpy(np.array([passes[x[2]][2][x[4]] for x in seq], np.float32).reshape(1, -1, 3))
        occ = rr.occupancy_activation(a)
        T = rr.occupancy_to_termination(occ, is_batch=False)
        out["depth"][r] = float(rr.render(T, z))
        out["colour"][r] = rr.render(T[..., None], c, dim=-2).numpy()[0]
        out["opacity"][r] = float(T.sum(-1))
        run = torch.cumsum(T[0], 0)
        hit = torch.nonzero(run >= 0.5)
        if len(hit):
            s = int(hit[0])
            out["zstar"][r], out["instance"][r], out["acc_at_surf"][r] = z[0, s], ids[seq[s][1]], run[s]
        else:
            out["acc_at_surf"][r] = run[-1]
    return out


def ref_render():
    rr = _refload.load("render_rays")
    T, boxes, ids, nets = ro.golden_scene()
    fns = reference_nets(nets)
    o, d = ro.rays(ro.GOLDEN_W, ro.GOLDEN_H, ro.GOLDEN_K, T)
    n = d.shape[0]
    src, ht, cnt, _ = ro.hit_table(boxes, o, d, ro.GOLDEN_NEAR, ro.GOLDEN_FAR)

    def evaluate(smp):
        alpha = np.zeros(len(smp["z"]), np.float32)
        col = np.zeros((len(smp["z"]), 3), np.float32)
        off = 0
        for s, m in enumerate(smp["totals"]):
            if m:
                alpha[off:off + m], col[off:off + m] = fns[s](smp["points"][off:off + m])
            off += m
        return alpha, col

    c = ro.samples(boxes, o, d, src, ht, cnt, ro.GOLDEN_NC)
    ca, cc = evaluate(c)
    r0 = reference_composite(n, src, ids, [(c, ca, cc)], rr)
    f = ro.samples(boxes, o, d, src, ht, cnt, ro.GOLDEN_NC, 1, r0["zstar"], ro.GOLDEN_EPS, ro.GOLDEN_NF)
    fa, fc = evaluate(f)
    r1 = reference_composite(n, src, ids, [(c, ca, cc), (f, fa, fc)], rr)
    return {"depth": r1["depth"], "colour": r1["colour"], "opacity": r1["opacity"], "instance": r1["instance"],
            "zstar": r0["zstar"], "acc_at_surf_coarse": r0["acc_at_surf"], "acc_at_surf": r1["acc_at_surf"],
            "hit_count": cnt, "n_coarse_points": np.int64(c["totals"].sum()), "n_fine_points": np.int64(f["totals"].sum())}


def main():
    np.savez_compressed(OUT, **ref_render())
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
