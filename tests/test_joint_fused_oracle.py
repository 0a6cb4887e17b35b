"""CPU checks of the fp16-faithful restatement of the joint map-and-pose step at hidden 32 (oracle/joint_fused_oracle.py):
with every rounding off its per-frame sums are the fp64 bundle-adjustment gradient of oracle/ba_oracle.py, the
whole-batch empty-mask rule of the mapping loss holds (central differences over the pose), a frame outside the table
contributes nothing, its weight gradients are fused_oracle.fused_step's, and the fp16 roundings stay near the exact
value."""
import numpy as np
import pytest
import torch

from oracle import ba_oracle as bo
from oracle import fused_oracle as fo
from oracle import joint_fused_oracle as jfo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo

NPD = 4                                            # rays per draw
SCALES = (1.3, 2.9, 3.7)                           # per object, not powers of two


def _pose(seed, deg=10.0, trans=0.1):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w / np.linalg.norm(w) * np.radians(deg))
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _case(B, R, S, seed, F=3):
    """fp64 weights, camera-frame samples with every mask count nonzero, an F-frame pose table and draws of NPD rays
    at frames (b + d) % F."""
    params = vo.init_params(B, 32, seed=seed, dtype=torch.float64)
    batch = vo.synthetic_batch(B, R, S, seed=seed + 1, n_cam2surf=S - 9 if S > 9 else 1, dtype=torch.float64)
    assert bool((fo.mask_counts(batch["sem"], batch["mask_depth"])[:, :3] > 0).all())
    scale = torch.tensor(SCALES[:B], dtype=torch.float32).double()
    d = torch.arange(R) // NPD
    frames = torch.stack([(b + d) % F for b in range(B)]).to(torch.int64)
    P = np.stack([_pose(seed + 10 + f) for f in range(F)])
    return params, scale, batch, frames, P


def _ba(params, scale, batch, frames, P):
    return bo.evaluate([{"params": params, "scale": scale, "batch": dict(batch, frames=frames)}], P)


@pytest.mark.parametrize("B,R,S", [(3, 24, 10), (2, 16, 14), (3, 20, 5), (1, 12, 17), (2, 8, 32)])
def test_rounding_off_is_the_ba_oracle(B, R, S):
    params, scale, batch, frames, P = _case(B, R, S, seed=B + S)
    out = jfo.evaluate(params, scale, batch, P, frames, rounding=jfo.ROUND_OFF)
    _, g, abs_sum, _ = _ba(params, scale, batch, frames, P)
    assert np.max(np.abs(out["grad"].numpy() - g)) <= 1e-10 * np.max(abs_sum)
    assert np.abs(g).max() > 1e-6 * np.max(abs_sum)


def _mapping_loss(params, scale, batch, frames, P, var):
    _, terms, _ = fo.fused_step(params, scale, dict(batch, pcs=jfo.world_points(P, frames, batch["pcs"], False)),
                                var=var, rounding=fo.ROUND_OFF)
    return float(terms[:, 3].sum())


def test_empty_mask_follows_the_whole_batch_rule():
    """Object 1 has no object pixel, so the mapping loss turns depth and colour off for every object (K11 keeps them on
    for the others): the rows are the gradient of that loss, shown by central differences over each frame's pose with
    the variance held, and they differ from K11's per-object rule."""
    params, scale, batch, frames, P = _case(3, 16, 10, seed=21)
    batch["sem"][1] = 0
    out = jfo.evaluate(params, scale, batch, P, frames, rounding=jfo.ROUND_OFF)
    assert torch.all(out["terms"][:, :2] == 0) and torch.all(out["terms"][:, 2] > 0)
    var = out["render"][1]
    h = 1e-7
    g = out["grad"].numpy()
    for f in range(P.shape[0]):
        fd = np.zeros(6)
        for i in range(6):
            e = np.zeros(6)
            e[i] = h
            Pp, Pm = P.copy(), P.copy()
            Pp[f], Pm[f] = to.retract(P[f], e), to.retract(P[f], -e)
            fd[i] = (_mapping_loss(params, scale, batch, frames, Pp, var) -
                     _mapping_loss(params, scale, batch, frames, Pm, var)) / (2 * h)
        assert np.allclose(fd, g[f], rtol=1e-5, atol=1e-5 * np.linalg.norm(g[f])), (f, fd, g[f])
    _, g_ba, _, _ = _ba(params, scale, batch, frames, P)
    assert np.abs(g_ba - g).max() > 0.1 * np.abs(g).max()


@pytest.mark.parametrize("rounding", ["off", "all"])
def test_frame_outside_the_table_contributes_nothing(rounding):
    """A draw whose frame is -1 keeps its camera-frame points, gets zero rows and adds nothing to any frame; the other
    rays' rows are those of a table in which that draw had a frame (the loss of a ray depends on its own pose only)."""
    rnd = jfo.ROUND_OFF if rounding == "off" else jfo.ROUND_ALL
    params, scale, batch, frames, P = _case(2, 16, 10, seed=5)
    bad = frames.clone()
    bad[1, NPD:2 * NPD] = -1
    ok = jfo.evaluate(params, scale, batch, P, frames, rounding=rnd)
    out = jfo.evaluate(params, scale, batch, P, bad, rounding=rnd)
    assert torch.all(out["rows"][1, NPD:2 * NPD] == 0)
    assert torch.equal(out["world"][1, NPD:2 * NPD], batch["pcs"][1, NPD:2 * NPD])
    keep = torch.ones(2, 16, dtype=torch.bool)
    keep[1, NPD:2 * NPD] = False
    scale_rows = float(ok["rows"].abs().max())
    assert torch.allclose(out["rows"][keep], ok["rows"][keep], rtol=0, atol=1e-12 * scale_rows)
    lost = ok["rows"][1, NPD:2 * NPD].sum(0)
    f = int(frames[1, NPD])
    want = ok["grad"].clone()
    want[f] -= lost
    assert torch.allclose(out["grad"], want, rtol=0, atol=1e-12 * scale_rows)


def test_weight_gradients_are_fused_steps():
    """The step is fused_step on the world points, bit for bit, and asking for its aux outputs changes nothing."""
    params, scale, batch, frames, P = _case(3, 20, 10, seed=8)
    out = jfo.evaluate(params, scale, batch, P, frames)
    wb = dict(batch, pcs=jfo.world_points(P, frames, batch["pcs"]))
    for aux in (None, {}):
        render, terms, grads = fo.fused_step(params, scale, wb, aux=aux)
        assert all(torch.equal(a, b) for a, b in zip(render, out["render"])) and torch.equal(terms, out["terms"])
        assert all(torch.equal(grads[k], out["grads"][k]) for k in vo.ALL_KEYS)
    assert torch.equal(out["dt"], aux["dt"]) and torch.equal(out["dproj"], aux["dproj"])


def test_rounding_stays_near_the_exact_value():
    """The fp16 stores move the rows, not by much (a bound on what the GPU bars mean): per frame relative to its
    norm, and summed per ray over sum |rows|."""
    params, scale, batch, frames, P = _case(3, 200, 10, seed=6)
    a = jfo.evaluate(params, scale, batch, P, frames, rounding=jfo.ROUND_OFF)
    b = jfo.evaluate(params, scale, batch, P, frames, rounding=jfo.ROUND_ALL)
    ga, gb = a["grad"].numpy(), b["grad"].numpy()
    e_f = max(np.abs(ga[f] - gb[f]).max() / np.linalg.norm(ga[f]) for f in range(P.shape[0]))
    e_r = float((a["rows"] - b["rows"]).abs().sum() / a["rows"].abs().sum())
    print(f"fp16 stores vs exact, 3 x 200 rays, H 32: per frame {e_f:.2e}, per ray {e_r:.2e}")
    assert e_f < 0.2 and e_r < 0.2
