"""Trajectory metrics (TUM RGB-D definitions) on the host: Umeyama alignment, ATE and RPE against closed forms."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from vmap_b200 import metrics


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _traj(n, seed):
    rng = np.random.default_rng(seed)
    return np.stack([_pose(Rotation.from_rotvec(rng.normal(size=3)).as_matrix(), rng.normal(size=3) * 2)
                     for _ in range(n)])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_align_recovers_a_rigid_transform(seed):
    P = _traj(50, seed)
    rng = np.random.default_rng(100 + seed)
    S = _pose(Rotation.from_rotvec(rng.normal(size=3)).as_matrix(), rng.normal(size=3) * 5)
    Q = S @ P
    assert np.max(np.abs(metrics.align_se3(P, Q) - S)) < 1e-12
    assert np.max(np.abs(metrics.align_se3(P[:, :3, 3], Q[:, :3, 3]) - S)) < 1e-12


def test_align_guards_against_reflection():
    P = _traj(40, 5)
    Q = P.copy()
    Q[:, :3, 3] *= np.array([1.0, 1.0, -1.0])          # a mirror image: the best proper rotation, not the reflection
    S = metrics.align_se3(P, Q)
    assert abs(np.linalg.det(S[:3, :3]) - 1.0) < 1e-12


def test_ate_aligned_and_unaligned():
    P = _traj(30, 7)
    S = _pose(Rotation.from_rotvec([0.3, -0.2, 0.5]).as_matrix(), [1.0, 2.0, -0.5])
    r = metrics.ate(P, S @ P, align=True)
    assert r["rmse"] < 1e-12 and r["max"] < 1e-12 and r["errors"].shape == (30,)
    off = np.array([0.3, -0.4, 1.2])
    Q = P.copy()
    Q[:, :3, 3] += off
    u = metrics.ate(P, Q, align=False)
    for k in ("rmse", "mean", "median", "max"):
        assert abs(u[k] - np.linalg.norm(off)) < 1e-12
    assert metrics.ate(P, Q, align=True)["rmse"] < 1e-12


def test_ate_statistics():
    gt = np.tile(np.eye(4), (4, 1, 1))
    est = gt.copy()
    est[:, 0, 3] = [0.0, 1.0, 2.0, 4.0]
    r = metrics.ate(est, gt, align=False)
    assert r["mean"] == pytest.approx(7 / 4) and r["median"] == pytest.approx(1.5) and r["max"] == 4.0
    assert r["rmse"] == pytest.approx(math.sqrt(21 / 4))


def test_rpe_invariant_to_a_global_rigid_transform():
    P, Q = _traj(25, 11), _traj(25, 12)
    S = _pose(Rotation.from_rotvec([0.1, 0.7, -0.3]).as_matrix(), [3.0, -1.0, 2.0])
    for d in (1, 3):
        a, b = metrics.rpe(P, Q, delta=d), metrics.rpe(S @ P, Q, delta=d)
        assert abs(a["trans_rmse"] - b["trans_rmse"]) < 1e-10
        assert abs(a["rot_rmse_deg"] - b["rot_rmse_deg"]) < 1e-8


def test_rpe_three_poses_by_hand():
    """GT moves 1 m along x per frame without turning; the estimate moves 1 m, then 1.5 m while turning 10 degrees about
    z.  Pair 0: no error.  Pair 1: E = rel_gt^-1 rel_est = translation (0.5, 0, 0) and a 10 degree rotation."""
    gt = np.stack([_pose(np.eye(3), [x, 0, 0]) for x in (0.0, 1.0, 2.0)])
    Rz = Rotation.from_euler("z", 10, degrees=True).as_matrix()
    est = np.stack([_pose(np.eye(3), [0, 0, 0]), _pose(np.eye(3), [1, 0, 0]), _pose(Rz, [2.5, 0, 0])])
    r = metrics.rpe(est, gt)
    assert np.allclose(r["trans_errors"], [0.0, 0.5], atol=1e-12)
    assert np.allclose(r["rot_errors_deg"], [0.0, 10.0], atol=1e-9)
    assert r["trans_rmse"] == pytest.approx(math.sqrt(0.25 / 2)) and r["rot_rmse_deg"] == pytest.approx(math.sqrt(50))
    r2 = metrics.rpe(est, gt, delta=2)
    assert np.allclose(r2["trans_errors"], [0.5]) and np.allclose(r2["rot_errors_deg"], [10.0])
