"""CPU checks of the several-group joint restatement (oracle/joint_groups_oracle.py: the vMAP objects and the
background model under one pose update), of the binding of vmb_joint_step_fused and of Slam's joint_impl guard."""
import os

import numpy as np
import pytest
import torch

from oracle import ba_oracle as bo
from oracle import joint_groups_oracle as jo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F, N_ITER = 4, 3
N_PIX = (6, 9)                                     # objects, background: rays per iteration


def _group(B, hidden, S, n_pix, seed, shift):
    params = vo.init_params(B, hidden, seed=seed, dtype=torch.float64)
    batch = vo.synthetic_batch(B, N_ITER * n_pix, S, seed=seed + 1, n_cam2surf=S - 9, dtype=torch.float64)
    d = torch.arange(N_ITER * n_pix) // 3                           # draws of 3 rays
    batch["frames"] = torch.stack([(b + shift + d) % F for b in range(B)]).to(torch.int64)
    return {"params": params, "scale": torch.full((B,), 3.0, dtype=torch.float64), "batch": batch}


def _case(seed=0):
    """Two hidden-32 objects (S 10) and a hidden-128 background (S 14), seen from the same four frames."""
    groups = [_group(2, 32, 10, N_PIX[0], seed, 0), _group(1, 128, 14, N_PIX[1], seed + 7, 1)]
    P = np.stack([np.eye(4)] * F)
    for f in range(F):
        P[f, :3, :3] = to.exp_so3_np([0.2 - 0.05 * f, -0.1 + 0.03 * f, 0.3])
        P[f, :3, 3] = [0.1 + 0.02 * f, -0.2, 0.05 - 0.01 * f]
    return groups, P


def test_pose_rates_zero_is_each_groups_mapping_step():
    groups, P = _case()
    out = jo.joint_groups(groups, P, [1, 2, 3], N_ITER, N_PIX, 1e-3, 0.013, 0.0, 0.0)
    assert np.array_equal(out["poses"][-1], P)
    total = np.zeros(N_ITER)
    for k, (g, n) in enumerate(zip(groups, N_PIX)):
        ens = vo.OracleEnsemble(g["params"], g["scale"], lr=1e-3, weight_decay=0.013)
        world = jo.world_batch(g["batch"], P)
        for it in range(N_ITER):
            total[it] += float(ens.step({kk: v[:, it * n:(it + 1) * n] for kk, v in world.items()}))
        for name, v in ens.params.items():
            assert torch.allclose(out["params"][k][name], v.detach(), rtol=1e-12, atol=1e-14), (k, name)
    assert np.allclose(out["losses"], total, rtol=1e-12, atol=0)


def test_weight_rate_zero_is_the_two_group_bundle_adjustment():
    groups, P = _case(seed=3)
    window = [0, 1, 2, 3]
    out = jo.joint_groups(groups, P, window, N_ITER, N_PIX, 0.0, 0.013, 0.01, 0.02)
    hist, _, grads = bo.bundle_adjust(groups, P, window, N_ITER, list(N_PIX), 0.01, 0.02)
    for g, p in zip(groups, out["params"]):
        for k, v in g["params"].items():
            assert torch.equal(p[k], v), k
    assert np.array_equal(out["poses"], hist)
    assert np.array_equal(out["pose_grads"], grads)
    assert not np.array_equal(hist[-1][1:], P[1:])                  # the poses did move


def test_held_frame_never_moves():
    groups, P = _case(seed=5)
    out = jo.joint_groups(groups, P, [0, 1, 2, 3], N_ITER, N_PIX, 1e-3, 0.013, 0.01, 0.01)
    assert np.array_equal(out["poses"][:, 0], np.broadcast_to(P[0], out["poses"][:, 0].shape))
    assert np.any(np.abs(out["pose_grads"][:, 0]) > 0)             # frame 0 has a gradient: held, not unseen
    assert not np.array_equal(out["poses"][-1][1:], P[1:])


def test_fused_joint_entry_is_declared_and_bound():
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    assert "int vmb_joint_step_fused(vmb_handle* h, const vmb_step_args* s, const vmb_ba_args* a, int group, " \
           "float* pcs_world_out,\n                         void* stream);" in src
    lib_src = open(os.path.join(ROOT, "vmap_b200", "_lib.py")).read()
    assert '"vmb_joint_step_fused"' in lib_src
    assert "L.vmb_joint_step_fused.argtypes = [_vp, C.POINTER(StepArgs), C.POINTER(BaArgs), C.c_int, _vp, _vp]" in lib_src


def test_slam_joint_impl_guards():
    from vmap_b200.cfg import Config, replica_room0_dict
    from vmap_b200.slam import Slam
    with pytest.raises(ValueError, match="iMAP"):
        Slam(Config(config_dict=replica_room0_dict(imap=True, device="cpu")), joint_poses=True, joint_impl="fused")
    with pytest.raises(ValueError, match='joint_impl="fused"'):
        Slam(Config(config_dict=replica_room0_dict(imap=False, device="cpu")), joint_poses=True)
    with pytest.raises(ValueError, match="joint_impl"):
        Slam(Config(config_dict=replica_room0_dict(imap=False, device="cpu")), joint_impl="tensor")
