"""CPU checks of the fp16-faithful layer-wise tracking restatement (oracle/track_lw_oracle.py): with every rounding off
it is the exact fp64 tracking rule of oracle/track_oracle.py, its per-frame gradients (pose per ray, as K11) equal
central differences of its own loss, and with the roundings on it stays near the exact gradient."""
import numpy as np
import pytest
import torch

from oracle import track_lw_oracle as tlo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo


def _case(hidden, B, R, S, seed):
    params = vo.init_params(B, hidden, seed=seed, dtype=torch.float64)
    batch = vo.synthetic_batch(B, R, S, seed=seed + 1, n_cam2surf=S - 9 if S > 9 else 1, dtype=torch.float64)
    return params, torch.full((B,), 2.0, dtype=torch.float64), batch


def _pose(seed, deg=20.0, trans=0.3):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w / np.linalg.norm(w) * np.radians(deg))
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


@pytest.mark.parametrize("hidden,B,R,S", [(64, 2, 11, 10), (128, 1, 9, 14), (256, 3, 7, 5), (64, 1, 5, 32)])
def test_rounding_off_is_the_tracking_oracle(hidden, B, R, S):
    params, scale, batch = _case(hidden, B, R, S, seed=hidden + S)
    T = _pose(hidden + B)
    out = tlo.evaluate(params, scale, batch, T, rounding=tlo.ROUND_OFF)
    loss, g, abs_sum, terms = to.evaluate([{"params": params, "scale": scale, "batch": batch}], T)
    assert np.max(np.abs(out["grad"][0].numpy() - g)) <= 1e-10 * np.max(abs_sum)
    # 1 - occ is sigmoid(-alpha) here (K10's rule) and 1 - sigmoid(alpha) there.  Where occ rounds near 1 the latter
    # cancels (absolute error ~1e-16 on a small transmittance), and the depth weight 1 / (sqrt(var) + 1e-4) amplifies
    # it: measured up to 1.4e-11 relative on the loss
    assert torch.allclose(out["terms"], terms[0], rtol=1e-9, atol=1e-11 * float(terms[0][:, 3].abs().max()))
    assert abs(out["loss"] - loss) <= 1e-9 * abs(loss)


def test_empty_masks_are_per_object_and_per_term():
    params, scale, batch = _case(64, 2, 12, 10, seed=3)
    batch["mask_depth"][1] = False
    T = _pose(4)
    out = tlo.evaluate(params, scale, batch, T, rounding=tlo.ROUND_OFF)
    _, g, abs_sum, terms = to.evaluate([{"params": params, "scale": scale, "batch": batch}], T)
    assert out["terms"][1, 0] == 0.0 and out["terms"][0, 0] > 0
    assert np.max(np.abs(out["grad"][0].numpy() - g)) <= 1e-10 * np.max(abs_sum)


def test_per_frame_gradients_match_central_differences():
    """A pose per ray (draws of 3 rays over three frames, one ray without a frame): the gradient of each frame equals
    central differences of the oracle's own loss, the depth term's variance held at the unperturbed poses."""
    params, scale, batch = _case(128, 2, 12, 10, seed=7)
    P = np.stack([_pose(10 + f, 10.0, 0.1) for f in range(3)])
    frames = torch.stack([(torch.arange(12) // 3 + b) % 3 for b in range(2)])
    frames[0, 5] = -1
    out = tlo.evaluate(params, scale, batch, P, frames, rounding=tlo.ROUND_OFF)
    assert torch.all(out["rows"][0, 5] == 0) and torch.all(out["ray_terms"][0, 5] == 0)
    h = 1e-7
    for f in range(3):
        fd = np.zeros(6)
        for i in range(6):
            e = np.zeros(6)
            e[i] = h
            Pp, Pm = P.copy(), P.copy()
            Pp[f], Pm[f] = to.retract(P[f], e), to.retract(P[f], -e)
            lp = tlo.evaluate(params, scale, batch, Pp, frames, rounding=tlo.ROUND_OFF, var=out["var"])["loss"]
            lm = tlo.evaluate(params, scale, batch, Pm, frames, rounding=tlo.ROUND_OFF, var=out["var"])["loss"]
            fd[i] = (lp - lm) / (2 * h)
        g = out["grad"][f].numpy()
        assert np.allclose(fd, g, rtol=1e-5, atol=1e-5 * np.linalg.norm(g)), (f, fd, g)


def test_rounding_stays_near_the_exact_gradient():
    """The fp16 stores move the gradient, not by much at a few hundred rays (a bound for the GPU bars' meaning)."""
    params, scale, batch = _case(256, 1, 200, 14, seed=5)
    T = _pose(6)
    a = tlo.evaluate(params, scale, batch, T, rounding=tlo.ROUND_OFF)
    b = tlo.evaluate(params, scale, batch, T, rounding=tlo.ROUND_ALL,
                     signs=None)
    err = np.abs(a["grad"][0].numpy() - b["grad"][0].numpy()).max() / np.linalg.norm(a["grad"][0].numpy())
    print(f"fp16 stores vs exact, 200 rays, H 256: {err:.2e}")
    assert err < 0.2
