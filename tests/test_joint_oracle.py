"""CPU checks of the joint map-and-pose restatement (oracle/joint_oracle.py) and of its C binding."""
import os

import numpy as np
import torch

from oracle import ba_oracle as bo
from oracle import joint_oracle as jo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F, N_ITER, N_PIX = 4, 3, 6


def _case(B=2, hidden=64, S=14, seed=0):
    params = vo.init_params(B, hidden, seed=seed, dtype=torch.float64)
    batch = vo.synthetic_batch(B, N_ITER * N_PIX, S, seed=seed + 1, n_cam2surf=S - 9, dtype=torch.float64)
    d = torch.arange(N_ITER * N_PIX) // 3                           # draws of 3 rays
    batch["frames"] = torch.stack([(b + d) % F for b in range(B)]).to(torch.int64)
    P = np.stack([np.eye(4)] * F)
    for f in range(F):
        P[f, :3, :3] = to.exp_so3_np([0.2 - 0.05 * f, -0.1 + 0.03 * f, 0.3])
        P[f, :3, 3] = [0.1 + 0.02 * f, -0.2, 0.05 - 0.01 * f]
    return params, torch.full((B,), 3.0, dtype=torch.float64), batch, P


def test_pose_rates_zero_is_the_mapping_step():
    params, scale, batch, P = _case()
    out = jo.joint(params, scale, batch, P, [1, 2, 3], N_ITER, N_PIX, 1e-3, 0.013, 0.0, 0.0)
    assert np.array_equal(out["poses"][-1], P)
    ens = vo.OracleEnsemble(params, scale, lr=1e-3, weight_decay=0.013)
    f = batch["frames"].clamp(min=0)
    Pt = torch.as_tensor(P)
    world = torch.einsum("brij,brsj->brsi", Pt[f, :3, :3], batch["pcs"]) + Pt[f, :3, 3][:, :, None, :]
    for it in range(N_ITER):
        sl = {k: v[:, it * N_PIX:(it + 1) * N_PIX] for k, v in batch.items() if k != "frames"}
        sl["pcs"] = world[:, it * N_PIX:(it + 1) * N_PIX]
        assert abs(float(ens.step(sl)) - out["losses"][it]) <= 1e-12 * abs(out["losses"][it])
    for k, v in ens.params.items():
        assert torch.allclose(out["params"][k], v.detach(), rtol=1e-12, atol=1e-14), k


def test_weight_rate_zero_is_bundle_adjustment():
    params, scale, batch, P = _case(seed=3)
    window = [0, 1, 2, 3]
    out = jo.joint(params, scale, batch, P, window, N_ITER, N_PIX, 0.0, 0.013, 0.01, 0.02)
    hist, _, grads = bo.bundle_adjust([{"params": params, "scale": scale, "batch": batch}], P, window, N_ITER,
                                      [N_PIX], 0.01, 0.02)
    for k, v in params.items():
        assert torch.equal(out["params"][k], v), k
    assert np.array_equal(out["poses"], hist)
    assert np.array_equal(out["pose_grads"], grads)
    assert not np.array_equal(hist[-1][1:], P[1:])                  # the poses did move


def test_frame_zero_never_moves():
    params, scale, batch, P = _case(B=1, hidden=128, seed=5)
    out = jo.joint(params, scale, batch, P, [0, 1, 2, 3], N_ITER, N_PIX, 1e-3, 0.013, 0.01, 0.01)
    assert np.array_equal(out["poses"][:, 0], np.broadcast_to(P[0], out["poses"][:, 0].shape))
    assert np.any(np.abs(out["pose_grads"][:, 0]) > 0)             # frame 0 has a gradient: held, not unseen
    assert not np.array_equal(out["poses"][-1][1:], P[1:])


def test_joint_entry_is_declared_and_bound():
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    assert "int vmb_joint_step_lw(vmb_handle* h, const vmb_step_args* s, const vmb_ba_args* a, int group, " \
           "float* pcs_world_out,\n                      void* stream);" in src
    lib_src = open(os.path.join(ROOT, "vmap_b200", "_lib.py")).read()
    assert '"vmb_joint_step_lw"' in lib_src
    assert "L.vmb_joint_step_lw.argtypes = [_vp, C.POINTER(StepArgs), C.POINTER(BaArgs), C.c_int, _vp, _vp]" in lib_src


def test_slam_refuses_joint_poses_outside_imap_mode():
    import pytest
    from vmap_b200.cfg import Config, replica_room0_dict
    from vmap_b200.slam import Slam
    with pytest.raises(ValueError, match="hidden-32"):
        Slam(Config(config_dict=replica_room0_dict(imap=False, device="cpu")), joint_poses=True)
