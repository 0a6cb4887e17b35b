"""CPU checks of the fp16-faithful restatement of the fused hidden-32 tracking step (oracle/track_fused_oracle.py): with
every rounding off it is the exact fp64 tracking rule of oracle/track_oracle.py, its gradient equals central
differences of its own loss, its BA rows with every ray at one frame are the track flavour, and its pose_point
restatement is the kernel's fp32 arithmetic bit for bit."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import track_fused_oracle as tfo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo


def _case(B, R, S, seed):
    params = vo.init_params(B, 32, seed=seed, dtype=torch.float64)
    batch = vo.synthetic_batch(B, R, S, seed=seed + 1, n_cam2surf=S - 9 if S > 9 else 1, dtype=torch.float64)
    return params, torch.full((B,), 2.0, dtype=torch.float64), batch


def _pose(seed, deg=20.0, trans=0.3):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w / np.linalg.norm(w) * np.radians(deg))
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


@pytest.mark.parametrize("B,R,S", [(3, 11, 10), (1, 9, 14), (2, 7, 5), (1, 5, 32)])
def test_rounding_off_is_the_tracking_oracle(B, R, S):
    params, scale, batch = _case(B, R, S, seed=B + S)
    T = _pose(B + R)
    out = tfo.evaluate(params, scale, batch, T, rounding=tfo.ROUND_OFF)
    loss, g, abs_sum, terms = to.evaluate([{"params": params, "scale": scale, "batch": batch}], T)
    assert np.max(np.abs(out["grad"][0].numpy() - g)) <= 1e-10 * np.max(abs_sum)
    # 1 - occ is sigmoid(-alpha) here and 1 - sigmoid(alpha) there (see test_track_lw_oracle): 1e-9 on the loss
    assert torch.allclose(out["terms"], terms[0], rtol=1e-9, atol=1e-11 * float(terms[0][:, 3].abs().max()))
    assert abs(out["loss"] - loss) <= 1e-9 * abs(loss)


def test_empty_masks_are_per_object_and_per_term():
    params, scale, batch = _case(2, 12, 10, seed=3)
    batch["mask_depth"][1] = False
    T = _pose(4)
    out = tfo.evaluate(params, scale, batch, T, rounding=tfo.ROUND_OFF)
    _, g, abs_sum, _ = to.evaluate([{"params": params, "scale": scale, "batch": batch}], T)
    assert out["terms"][1, 0] == 0.0 and out["terms"][0, 0] > 0
    assert np.max(np.abs(out["grad"][0].numpy() - g)) <= 1e-10 * np.max(abs_sum)


def test_gradient_matches_central_differences():
    """The track flavour's gradient equals central differences of the restatement's own loss (variance held)."""
    params, scale, batch = _case(2, 10, 10, seed=7)
    T = _pose(11, 10.0, 0.1)
    out = tfo.evaluate(params, scale, batch, T, rounding=tfo.ROUND_OFF)
    h = 1e-7
    fd = np.zeros(6)
    for i in range(6):
        e = np.zeros(6)
        e[i] = h
        lp = tfo.evaluate(params, scale, batch, to.retract(T, e), rounding=tfo.ROUND_OFF, var=out["var"])["loss"]
        lm = tfo.evaluate(params, scale, batch, to.retract(T, -e), rounding=tfo.ROUND_OFF, var=out["var"])["loss"]
        fd[i] = (lp - lm) / (2 * h)
    g = out["grad"][0].numpy()
    assert np.allclose(fd, g, rtol=1e-5, atol=1e-5 * np.linalg.norm(g)), (fd, g)


@pytest.mark.parametrize("rounding", ["off", "all"])
def test_ba_rows_at_one_frame_are_the_track_flavour(rounding):
    """Every ray at frame 1 of a three-pose table: the per-ray rows summed are the track flavour at that pose."""
    rnd = tfo.ROUND_OFF if rounding == "off" else tfo.ROUND_ALL
    params, scale, batch = _case(2, 12, 10, seed=9)
    P = np.stack([_pose(20 + f, 10.0, 0.1) for f in range(3)])
    ba = tfo.evaluate(params, scale, batch, P, torch.ones(2, 12, dtype=torch.int64), rounding=rnd)
    tr = tfo.evaluate(params, scale, batch, P[1], rounding=rnd)
    assert torch.equal(ba["rows"], tr["rows"]) and torch.equal(ba["ray_terms"], tr["ray_terms"])
    assert torch.allclose(ba["rows"].sum((0, 1)), tr["grad"][0], rtol=1e-12, atol=1e-12 * float(tr["abs_sum"].max()))
    assert torch.all(ba["grad"][0] == 0) and torch.all(ba["grad"][2] == 0)


def test_frame_outside_the_table_contributes_nothing():
    params, scale, batch = _case(2, 9, 10, seed=12)
    frames = torch.zeros(2, 9, dtype=torch.int64)
    frames[1, 4] = -1
    out = tfo.evaluate(params, scale, batch, _pose(13), frames)
    assert torch.all(out["rows"][1, 4] == 0) and torch.all(out["ray_terms"][1, 4] == 0)
    assert torch.all(out["t"][1, 4] == 0)


def test_rounding_stays_near_the_exact_gradient():
    """The fp16 stores move the gradient, not by much at a few hundred rays (a bound for the GPU bars' meaning)."""
    params, scale, batch = _case(2, 200, 10, seed=5)
    T = _pose(6)
    a = tfo.evaluate(params, scale, batch, T, rounding=tfo.ROUND_OFF)
    b = tfo.evaluate(params, scale, batch, T, rounding=tfo.ROUND_ALL)
    err = np.abs(a["grad"][0].numpy() - b["grad"][0].numpy()).max() / np.linalg.norm(a["grad"][0].numpy())
    print(f"fp16 stores vs exact, 2 x 200 rays, H 32: {err:.2e}")
    assert err < 0.2


# ---- pose_point: a float32 emulation with exact fma ----------------------------------------------------------------

def _round32(x: Fraction) -> np.float32:
    """x rounded to the nearest float32, ties to even (exact: Fraction arithmetic)."""
    f = np.float32(float(x))
    best = None
    for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        d = abs(Fraction(float(c)) - x)
        key = (d, int(np.frombuffer(c.tobytes(), np.uint32)[0]) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def _pose_point32(T, q, sc):
    """k_track.cuh pose_point, one fp32 operation at a time: fmaf(T2, qz, fmaf(T1, qy, T0 * qx)) + T3, then / scale."""
    F = lambda v: Fraction(float(v))                       # noqa: E731
    T32 = [np.float32(v) for v in np.asarray(T, np.float64).reshape(16)]
    out = []
    for r in range(3):
        x = _round32(F(T32[4 * r]) * F(q[0]))
        x = _round32(F(T32[4 * r + 1]) * F(q[1]) + F(x))
        x = _round32(F(T32[4 * r + 2]) * F(q[2]) + F(x))
        x = _round32(F(x) + F(T32[4 * r + 3]))
        out.append(_round32(F(x) / F(np.float32(sc))))
    return np.array(out, np.float32)


@pytest.mark.parametrize("sc", [2.0, 0.37, 5.0])
def test_pose_point_is_the_kernels_fp32_arithmetic(sc):
    rng = np.random.default_rng(int(sc * 100))
    B, R, S = 2, 6, 7
    q = torch.from_numpy(rng.uniform(-4, 4, (B, R, S, 3)).astype(np.float32)).double()
    P = np.stack([_pose(30 + f, 40.0, 2.0) for f in range(2)])
    frames = torch.from_numpy(rng.integers(0, 2, (B, R)))
    t, _ = tfo.posed_points(P, frames, q, sc)
    for b in range(B):
        for r in range(R):
            for s in range(S):
                want = _pose_point32(P[int(frames[b, r])], q[b, r, s].numpy(), sc)
                got = t[b, r, s].numpy().astype(np.float32)
                assert np.array_equal(got, want), (b, r, s, got, want)
