"""numpy restatement of the view renderer (vmap_b200/render.py, rule in vmap_b200/csrc/k_render.cuh).

TEST INFRASTRUCTURE ONLY.  The geometry (rays, slab test, sample z and points, fine positions) is fp64 in the operation
order the kernel header writes down; numpy rounds every operation on its own, so hit tables, z and points are bitwise
what the kernels compute.  The network is ``oracle/vmap_oracle.forward`` (fp32, CPU) through a callback, and
compositing is fp32 in the merged (z, source, pass, k) order.
"""
from __future__ import annotations

from typing import Callable, Dict

import numpy as np
import torch

MAX_HITS = 16


def rays(W: int, H: int, K, T, ray0: int = 0, n: int = None):
    """(o [3], d [n,3]) fp64 of rays ray0 .. ray0+n (pixel (u, v) = ray u*H + v)."""
    n = W * H - ray0 if n is None else n
    g = np.arange(ray0, ray0 + n, dtype=np.int64)
    u, v = (g // H).astype(np.float64), (g % H).astype(np.float64)
    K, T = np.asarray(K, np.float64), np.asarray(T, np.float64)
    dcx = (u - K[0, 2]) / K[0, 0]
    dcy = (v - K[1, 2]) / K[1, 1]
    d = np.stack([(T[j, 0] * dcx + T[j, 1] * dcy) + T[j, 2] for j in range(3)], 1)
    return T[:3, 3].copy(), d


def slab(boxes: np.ndarray, o, d, near: float, far: float):
    """(hit [n,S], t0 [n,S], t1 [n,S]) of every ray against every box row (center, R row-major, half, offset)."""
    n, S = d.shape[0], boxes.shape[0]
    t0 = np.full((n, S), float(near))
    t1 = np.full((n, S), float(far))
    ok = np.ones((n, S), bool)
    c, R, h = boxes[:, 0:3], boxes[:, 3:12].reshape(S, 3, 3), boxes[:, 12:15]
    q = o[None, :] - c                                                      # [S,3]
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(3):
            op = (R[:, 0, i] * q[:, 0] + R[:, 1, i] * q[:, 1]) + R[:, 2, i] * q[:, 2]               # [S]
            dp = (R[None, :, 0, i] * d[:, 0:1] + R[None, :, 1, i] * d[:, 1:2]) + R[None, :, 2, i] * d[:, 2:3]
            par = dp == 0.0
            ok &= ~(par & ~(np.abs(op) <= h[:, i])[None, :])
            a = (-h[None, :, i] - op[None, :]) / dp
            b = (h[None, :, i] - op[None, :]) / dp
            lo, hi = np.minimum(a, b), np.maximum(a, b)
            t0 = np.where(par, t0, np.maximum(t0, lo))
            t1 = np.where(par, t1, np.minimum(t1, hi))
    t0, t1 = t0 + 0.0, t1 + 0.0                                             # -0.0 -> +0.0, as the kernel
    return ok & (t0 < t1), t0, t1


def hit_table(boxes, o, d, near, far):
    """hit_src [n,16] (-1 past the count), hit_t [n,16,2], hit_count [n], overflow (rays with > 16 hits)."""
    hit, t0, t1 = slab(boxes, o, d, near, far)
    n = d.shape[0]
    key = np.where(hit, t0, np.inf)
    order = np.argsort(key, axis=1, kind="stable")[:, :MAX_HITS]          # (t0, source) order
    cnt_all = hit.sum(1)
    cnt = np.minimum(cnt_all, MAX_HITS)
    S = boxes.shape[0]
    k = min(MAX_HITS, S)
    src = np.full((n, MAX_HITS), -1, np.int32)
    ht = np.zeros((n, MAX_HITS, 2))
    valid = np.arange(k)[None, :] < cnt[:, None]
    src[:, :k] = np.where(valid, order[:, :k], -1)
    rows = np.arange(n)[:, None]
    ht[:, :k, 0] = np.where(valid, t0[rows, order[:, :k]], 0.0)
    ht[:, :k, 1] = np.where(valid, t1[rows, order[:, :k]], 0.0)
    return src, ht, cnt.astype(np.int32), int((cnt_all > MAX_HITS).sum())


def fine_positions(zstar: np.ndarray, eps: float, n_fine: int):
    """[n, n_fine] fp64 positions of the fine band around z* (fp32 input)."""
    zs = zstar.astype(np.float32).astype(np.float64)
    k = np.arange(n_fine, dtype=np.float64) + 0.5
    return (zs[:, None] - eps) + k[None, :] * ((eps + eps) / n_fine)


def samples(boxes, o, d, src, ht, cnt, n_coarse: int, pass_: int = 0, zstar=None, eps=0.1, n_fine=0):
    """One pass's samples, source-major: points [N,3] f32, z [N] f32, base [n,16], totals [S], and per sample
    (ray, slot, k) for compositing."""
    n, S = d.shape[0], boxes.shape[0]
    zk_rows, meta, counts = [], [], np.zeros((n, MAX_HITS), np.int64)
    if pass_ == 1:
        fy = fine_positions(zstar, eps, n_fine)
    for r in range(n):
        for i in range(cnt[r]):
            t0, t1 = ht[r, i]
            if pass_ == 0:
                w = (t1 - t0) / n_coarse
                zk = t0 + (np.arange(n_coarse, dtype=np.float64) + 0.5) * w
                ks = np.arange(n_coarse)
            else:
                if not zstar[r] >= 0:
                    continue
                ks = np.nonzero((t0 <= fy[r]) & (fy[r] <= t1))[0]
                zk = fy[r, ks]
            counts[r, i] = len(ks)
            if len(ks):
                zk_rows.append((src[r, i], r, i, zk, ks))
    totals = np.zeros(S, np.int64)
    for s, r, i, zk, ks in zk_rows:
        totals[s] += len(ks)
    zk_rows.sort(key=lambda x: (x[0], x[1]))
    base = np.zeros((n, MAX_HITS), np.int64)
    pts, zs, meta = [], [], []
    off = 0
    for s, r, i, zk, ks in zk_rows:
        base[r, i] = off
        p = o[None, :] + zk[:, None] * d[r][None, :]
        pts.append(p.astype(np.float32) - boxes[s, 15:18].astype(np.float32)[None, :])
        zs.append(zk.astype(np.float32))
        meta.append(np.stack([np.full(len(ks), r), np.full(len(ks), i), ks], 1))
        off += len(ks)
    cat = lambda xs, shp, dt: np.concatenate(xs) if xs else np.zeros(shp, dt)
    return {"points": cat(pts, (0, 3), np.float32), "z": cat(zs, (0,), np.float32), "base": base, "totals": totals,
            "counts": counts, "meta": cat(meta, (0, 3), np.int64)}


def composite(n: int, src, obj_id, passes):
    """fp32 front-to-back compositing of the merged samples of each ray.  ``passes`` = list of (samples dict, alpha
    [N], colour [N,3]) in pass order.  Returns depth, colour, opacity, instance, zstar (-1 = none), surf, and the running
    opacity at the surface sample (for tie-aware comparisons)."""
    per_ray = [[] for _ in range(n)]
    for p, (smp, alpha, col) in enumerate(passes):
        for j, (r, i, k) in enumerate(smp["meta"]):
            per_ray[r].append((float(smp["z"][j]), int(src[r, i]), p, int(k), j))
    out = {"depth": np.zeros(n, np.float32), "colour": np.zeros((n, 3), np.float32),
           "opacity": np.zeros(n, np.float32), "instance": np.full(n, -1, np.int32),
           "zstar": np.full(n, -1.0, np.float32), "surf": np.full(n, -1, np.int32), "acc_at_surf": np.full(n, np.nan)}
    one, tiny = np.float32(1.0), np.float32(1e-10)
    for r in range(n):
        seq = sorted(per_ray[r])
        if not seq:
            continue
        z = np.array([x[0] for x in seq], np.float32)
        a = np.array([passes[x[2]][1][x[4]] for x in seq], np.float32)
        c = np.array([passes[x[2]][2][x[4]] for x in seq], np.float32).reshape(-1, 3)
        occ = (one / (one + np.exp(-a))).astype(np.float32)
        free = np.concatenate([[one], ((one - occ) + tiny)[:-1]]).astype(np.float32)
        T = (occ * np.cumprod(free, dtype=np.float32)).astype(np.float32)
        run = np.cumsum(T, dtype=np.float32)
        out["depth"][r] = np.sum(T * z, dtype=np.float32)
        out["colour"][r] = np.sum(T[:, None] * c, axis=0, dtype=np.float32)
        out["opacity"][r] = run[-1]
        hit = np.nonzero(run >= np.float32(0.5))[0]
        if len(hit):
            s = int(hit[0])
            out["surf"][r], out["zstar"][r], out["acc_at_surf"][r] = s, z[s], run[s]
            out["instance"][r] = obj_id[seq[s][1]]
        else:
            out["acc_at_surf"][r] = run[-1]
    return out


def render(boxes, obj_id, net: Callable, W, H, K, T, n_coarse=32, n_fine=16, eps=0.1, near=0.0, far=1e4,
           zstar_inject=None) -> Dict[str, np.ndarray]:
    """The whole view.  ``net(source, points f32 [N,3]) -> (alpha [N], colour [N,3])`` fp32."""
    boxes = np.asarray(boxes, np.float64)
    o, d = rays(W, H, K, T)
    n = d.shape[0]
    src, ht, cnt, ovf = hit_table(boxes, o, d, near, far)

    def evaluate(smp):
        alpha = np.zeros(len(smp["z"]), np.float32)
        col = np.zeros((len(smp["z"]), 3), np.float32)
        off = 0
        for s, m in enumerate(smp["totals"]):
            if m:
                alpha[off:off + m], col[off:off + m] = net(s, smp["points"][off:off + m])
            off += m
        return alpha, col

    c = samples(boxes, o, d, src, ht, cnt, n_coarse)
    ca, cc = evaluate(c)
    r0 = composite(n, src, obj_id, [(c, ca, cc)])
    out = {"hit_src": src, "hit_t": ht, "hit_count": cnt, "overflow": ovf, "coarse": c, "coarse_comp": r0}
    if n_fine == 0:
        final = r0
    else:
        zs = r0["zstar"] if zstar_inject is None else zstar_inject
        f = samples(boxes, o, d, src, ht, cnt, n_coarse, 1, zs, eps, n_fine)
        fa, fc = evaluate(f)
        final = composite(n, src, obj_id, [(c, ca, cc), (f, fa, fc)])
        out["fine"] = f
    out.update({k: final[k] for k in ("depth", "colour", "opacity", "instance", "acc_at_surf")})
    out["zstar"] = r0["zstar"]
    return out


def oracle_net(params: Dict[str, torch.Tensor], scale: float):
    """A ``net`` callback for one source from its [1, ...] stacked parameters (vmap_oracle.forward, fp32 CPU)."""
    from oracle import vmap_oracle as vo

    def f(pts: np.ndarray):
        with torch.no_grad():
            a, c = vo.forward(params, torch.tensor([scale], dtype=torch.float32),
                              torch.from_numpy(np.ascontiguousarray(pts, np.float32)).view(1, -1, 1, 3))
        return a.reshape(-1).numpy(), c.reshape(-1, 3).numpy()
    return f


GOLDEN_W, GOLDEN_H, GOLDEN_NC, GOLDEN_NF, GOLDEN_EPS, GOLDEN_NEAR, GOLDEN_FAR = 48, 36, 8, 4, 0.1, 0.05, 6.0
GOLDEN_K = np.array([[40.0, 0, 23.5], [0, 40.0, 17.5], [0, 0, 1]])


def golden_scene():
    """The scene of tests/golden/ref_render.npz: a 48 x 36 view, hidden-32 objects and one hidden-128 source (id 0) in
    five boxes (one containing the camera, two overlapping -- one of them the hidden-128 --, one behind the camera,
    one off-screen).  Returns
    (T_wc, boxes [5,18], obj_id [5], per-source (params [1,...] fp32, scale))."""
    from oracle import vmap_oracle as vo
    T = np.eye(4)
    T[:3, 3] = [0.1, -0.05, 0.0]
    a = 0.4
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    boxes = np.stack([
        np.concatenate([[0.1, -0.05, 0.2], np.eye(3).reshape(9), [0.5, 0.4, 0.6], [0, 0, 0]]),      # camera inside
        np.concatenate([[0.2, 0.1, 2.0], R.reshape(9), [0.5, 0.4, 0.5], [0, 0, 0]]),               # overlapping pair
        np.concatenate([[-0.1, 0.0, 2.4], R.T.reshape(9), [0.4, 0.5, 0.6], [0, 0, 0]]),
        np.concatenate([[0.0, 0.0, -2.0], np.eye(3).reshape(9), [0.5, 0.5, 0.5], [0, 0, 0]]),     # behind
        np.concatenate([[9.0, 0.0, 2.0], np.eye(3).reshape(9), [0.5, 0.5, 0.5], [0, 0, 0]]),      # off-screen
    ])
    ids = np.array([3, 5, 0, 9, 8], np.int32)
    p32 = vo.init_params(3, 32, seed=11)
    p128 = vo.init_params(1, 128, seed=12)
    nets = []
    for s in range(5):
        src, row = (p128, 0) if s == 2 else (p32, s % 3)
        p = {k: v[row:row + 1].clone() for k, v in src.items()}
        if s == 0:                                     # the box around the camera is nearly empty space
            p["out_alpha.weight"] *= 0.1
            p["out_alpha.bias"].fill_(-0.6)
        else:                                          # decisive occupancies: few rays near the 0.5 threshold
            p["out_alpha.weight"] *= 8.0
            p["out_alpha.bias"] += 0.1
        nets.append((p, 3.0 if s == 2 else 2.0))
    return T, boxes, ids, nets


def golden_render():
    """The oracle on the golden scene (vmap_oracle.forward networks)."""
    T, boxes, ids, nets = golden_scene()
    fns = [oracle_net(p, sc) for p, sc in nets]
    return render(boxes, ids, lambda s, pts: fns[s](pts), GOLDEN_W, GOLDEN_H, GOLDEN_K, T, GOLDEN_NC, GOLDEN_NF,
                  GOLDEN_EPS, GOLDEN_NEAR, GOLDEN_FAR)
