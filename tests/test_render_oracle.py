"""CPU checks of the view-rendering oracle (oracle/render_oracle.py): slab-test geometry against a dense march, the
edge cases of the rule in k_render.cuh, sample placement, and metrics.view_metrics on hand-computed cases."""
import math

import numpy as np
import pytest
import torch

from oracle import render_oracle as ro

K = np.array([[40.0, 0, 23.5], [0, 40.0, 17.5], [0, 0, 1]])


def box(c, half, R=None, off=(0, 0, 0)):
    R = np.eye(3) if R is None else np.asarray(R)
    return np.concatenate([np.asarray(c, float), R.reshape(9), np.asarray(half, float), np.asarray(off, float)])


def rot(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def pose(seed):
    T = np.eye(4)
    T[:3, :3] = rot(seed + 100) @ np.diag([1, 1, 1])
    T[:3, 3] = np.random.default_rng(seed).normal(size=3) * 0.3
    return T


def inside(b, p, tol):
    c, R, h = b[0:3], b[3:12].reshape(3, 3), b[12:15]
    return np.all(np.abs((p - c) @ R) <= h + tol, axis=-1)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_samples_inside_box_and_depth_range(seed):
    rng = np.random.default_rng(seed)
    T = pose(seed)
    boxes = np.stack([box(T[:3, 3] + T[:3, :3] @ rng.normal([0, 0, 2.5], 0.6), rng.uniform(0.2, 0.6, 3), rot(seed * 7 + i))
                      for i in range(5)])
    o, d = ro.rays(48, 36, K, T)
    near, far = 0.1, 4.0
    src, ht, cnt, _ = ro.hit_table(boxes, o, d, near, far)
    smp = ro.samples(boxes, o, d, src, ht, cnt, 8)
    assert smp["points"].shape[0] == cnt.sum() * 8 > 0
    for j in range(0, len(smp["z"]), 7):
        r, i, k = smp["meta"][j]
        z = float(smp["z"][j])
        w = (ht[r, i, 1] - ht[r, i, 0]) / 8
        zk = ht[r, i, 0] + (k + 0.5) * w
        assert near <= zk <= far
        assert inside(boxes[src[r, i]], o + zk * d[r], 1e-9)
        assert z == np.float32(zk)


@pytest.mark.parametrize("seed", [3, 4])
def test_slab_agrees_with_dense_march(seed):
    rng = np.random.default_rng(seed)
    b = box(rng.normal(size=3) * 0.2 + [0, 0, 2], rng.uniform(0.2, 0.7, 3), rot(seed))
    o = rng.normal(size=3) * 0.1
    d = rng.normal(size=(400, 3)) * [0.4, 0.4, 0.1] + [0, 0, 1]
    near, far = 0.05, 5.0
    hit, t0, t1 = ro.slab(b[None], o, d, near, far)
    ts = np.linspace(near, far, 4001)
    c, R, h = b[0:3], b[3:12].reshape(3, 3), b[12:15]
    for r in range(len(d)):
        margin = np.min(h - np.abs((o[None] + ts[:, None] * d[r][None] - c) @ R), axis=1)
        marched = margin > 1e-9                             # inside, not within 1e-9 of a face
        if marched.any():
            assert hit[r, 0], r
            assert t0[r, 0] <= ts[marched][0] and ts[marched][-1] <= t1[r, 0]
        elif hit[r, 0]:                                     # a hit thinner than the march step: its midpoint is inside
            mid = o + 0.5 * (t0[r, 0] + t1[r, 0]) * d[r]
            assert np.min(h - np.abs((mid - c) @ R)) >= -1e-9


def test_camera_inside_box_starts_at_near():
    b = box([0, 0, 0], [1, 1, 1])
    o, d = ro.rays(4, 3, K, np.eye(4))
    hit, t0, t1 = ro.slab(b[None], o, d, 0.2, 10.0)
    assert hit.all() and (t0 == 0.2).all() and (t1 > 0.2).all()


def test_ray_parallel_to_face():
    o = np.zeros(3)
    d = np.array([[0.0, 0.0, 1.0]])
    inside_slab = box([0.3, 0, 3], [0.5, 0.5, 0.5])     # |o'_x| = 0.3 <= 0.5
    outside_slab = box([0.7, 0, 3], [0.5, 0.5, 0.5])    # |o'_x| = 0.7 > 0.5
    on_face = box([0.5, 0, 3], [0.5, 0.5, 0.5])         # |o'_x| = 0.5: closed slab
    hit, t0, t1 = ro.slab(np.stack([inside_slab, outside_slab, on_face]), o, d, 0.0, 10.0)
    assert hit[0].tolist() == [True, False, True]
    assert t0[0, 0] == 2.5 and t1[0, 0] == 3.5


def test_box_behind_camera_no_hit():
    o, d = ro.rays(6, 5, K, np.eye(4))
    hit, _, _ = ro.slab(box([0, 0, -3], [1, 1, 1])[None], o, d, 0.0, 10.0)
    assert not hit.any()


def test_overflow_keeps_nearest_16():
    boxes = np.stack([box([0, 0, 1.0 + 0.5 * i], [0.2, 0.2, 0.2]) for i in range(20)][::-1])   # far first
    o, d = np.zeros(3), np.array([[0.0, 0.0, 1.0], [5.0, 0.0, 1.0]])
    src, ht, cnt, ovf = ro.hit_table(boxes, o, d, 0.0, 100.0)
    assert ovf == 1 and cnt.tolist() == [16, 0]
    assert src[0].tolist() == list(range(19, 3, -1))
    assert np.all(np.diff(ht[0, :, 0]) > 0)
    # equal t0: ties by source index
    same = np.stack([box([0, 0, 2], [0.2, 0.2, 0.2])] * 3)
    src, ht, cnt, _ = ro.hit_table(same, o, d[:1], 0.0, 100.0)
    assert src[0, :3].tolist() == [0, 1, 2]


def test_composite_rule_by_hand():
    # two boxes on one ray, constant networks: occupancy 0.5 in the near box, ~1 in the far box
    boxes = np.stack([box([0, 0, 2], [0.5, 0.5, 0.5]), box([0, 0, 4], [0.5, 0.5, 0.5])])
    ids = np.array([7, 9], np.int32)

    def net(s, pts):
        n = len(pts)
        return (np.full(n, 0.0 if s == 0 else 50.0, np.float32),
                np.tile(np.array([[1, 0, 0]] if s == 0 else [[0, 1, 0]], np.float32), (n, 1)))
    out = ro.render(boxes, ids, net, 1, 1, np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1]]), np.eye(4),
                    n_coarse=2, n_fine=0, near=0.0, far=10.0)
    # samples z = 1.75, 2.25 (occ 0.5) then 3.75, 4.25 (occ 1): T = 0.5, 0.25, 0.25, 0
    assert out["instance"][0] == 7 and out["zstar"][0] == np.float32(1.75)
    assert math.isclose(float(out["opacity"][0]), 1.0, rel_tol=1e-6)
    assert math.isclose(float(out["depth"][0]), 0.5 * 1.75 + 0.25 * 2.25 + 0.25 * 3.75, rel_tol=1e-6)
    assert np.allclose(out["colour"][0], [0.75, 0.25, 0.0], rtol=1e-6)


def test_view_metrics_by_hand():
    from vmap_b200.metrics import view_metrics
    gt = torch.zeros(4, 2, 3, dtype=torch.float64)
    col = gt.clone()
    col[0, 0] = 0.1                                        # one pixel off by 0.1 in every channel
    gd = torch.tensor([[1.0, 2.0], [0.0, 1.0], [1.0, 1.0], [1.0, 1.0]])
    d = gd.clone()
    d[0, 1] = 2.5
    d[1, 0] = 9.0                                          # gt 0: ignored
    inst = torch.tensor([[1, 1], [0, 0], [2, 2], [2, 2]])
    m = view_metrics(col, d, gt, gd, inst)
    assert math.isclose(m["psnr"], -10 * math.log10(0.01 / 8), rel_tol=1e-12)
    assert math.isclose(m["depth_l1"], 0.5 / 7, rel_tol=1e-12)
    assert m["obj_psnr"] == float("inf")                  # instance 2 is exact
    m2 = view_metrics(col, d, gt, gd, torch.tensor([[1, 1], [0, 0], [0, 0], [0, 0]]))
    assert math.isclose(m2["obj_psnr"], -10 * math.log10(0.01 / 2), rel_tol=1e-12)


def test_oracle_matches_reference_golden():
    """tests/golden/ref_render.npz: the reference's UniDirsEmbed / OccupancyMap / occupancy_to_termination / render on
    the oracle's samples (oracle/make_render_golden.py).  The oracle reproduces it with its own network and
    compositing: depth, colour and opacity to 1e-6 relative, instance and coarse z* exactly."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_render.npz"))
    out = ro.golden_render()
    assert np.array_equal(out["hit_count"], g["hit_count"])
    assert out["coarse"]["totals"].sum() == g["n_coarse_points"] and out["fine"]["totals"].sum() == g["n_fine_points"]
    assert (g["instance"] >= 0).sum() > 50 and len(set(g["instance"].tolist())) >= 3
    assert np.array_equal(out["zstar"], g["zstar"])
    assert np.array_equal(out["instance"], g["instance"])
    for k in ("depth", "colour", "opacity"):
        a, b = out[k].astype(np.float64), g[k].astype(np.float64)
        assert np.linalg.norm(a - b) <= 1e-6 * np.linalg.norm(b), k
