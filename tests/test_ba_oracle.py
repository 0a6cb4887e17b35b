"""CPU checks of the bundle-adjustment restatement (oracle/ba_oracle.py) and of the K11 binding."""
import os
import re

import numpy as np
import torch

from oracle import ba_oracle as bo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 4


def _groups(frames_fn, seed=0):
    """Two groups (hidden 32 with two objects, hidden 64 with one), 12 rays each in draws of 3 rays."""
    out = []
    for hidden, B, S, sc in ((32, 2, 10, 2.0), (64, 1, 14, 5.0)):
        params = vo.init_params(B, hidden, seed=seed + hidden, dtype=torch.float64)
        batch = vo.synthetic_batch(B, 12, S, seed=seed + hidden + 1, n_cam2surf=S - 9, dtype=torch.float64)
        batch["frames"] = frames_fn(B, hidden)
        out.append({"params": params, "scale": torch.full((B,), sc, dtype=torch.float64), "batch": batch})
    return out


def _draws(B, hidden):
    """Draw d of object b is seen from frame (b + d + hidden) % F: frames shared across objects and groups."""
    d = torch.arange(12) // 3
    return torch.stack([(b + d + hidden) % F for b in range(B)]).to(torch.int64)


def _poses():
    P = np.stack([np.eye(4)] * F)
    for f in range(F):
        P[f, :3, :3] = to.exp_so3_np([0.2 - 0.05 * f, -0.1 + 0.03 * f, 0.3])
        P[f, :3, 3] = [0.1 + 0.02 * f, -0.2, 0.05 - 0.01 * f]
    return P


def test_one_pose_for_every_ray_equals_the_tracking_oracle():
    groups = _groups(lambda B, h: torch.zeros(B, 12, dtype=torch.int64))
    P = _poses()
    loss, g, abs_sum, terms = bo.evaluate(groups, P)
    tl, tg, tabs, tterms = to.evaluate(groups, P[0])
    assert abs(loss - tl) <= 1e-12 * abs(tl)
    assert np.max(np.abs(g[0] - tg)) <= 1e-12 * np.max(tabs)
    assert np.all(g[1:] == 0.0)
    assert np.allclose(abs_sum[0], tabs, rtol=1e-12, atol=0)
    for a, b in zip(terms, tterms):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-15)


def test_per_frame_gradients_match_central_differences():
    groups, P = _groups(_draws), _poses()
    loss, g, abs_sum, _ = bo.evaluate(groups, P)
    assert abs(loss - bo.loss_at(groups, P)) <= 1e-12 * abs(loss)
    h = 1e-8      # a ray of frame 1 sits within 1e-6 of an L1 kink here; at 1e-8 the differences are past it
    for f in range(F):
        fd = np.zeros(6)
        for i in range(6):
            e = np.zeros(6)
            e[i] = h
            Pp, Pm = P.copy(), P.copy()
            Pp[f], Pm[f] = to.retract(P[f], e), to.retract(P[f], -e)
            fd[i] = (bo.loss_at(groups, Pp, var_poses=P) - bo.loss_at(groups, Pm, var_poses=P)) / (2 * h)
        # var is detached, so the differences hold it at the unperturbed poses (as test_track_oracle does for K10)
        assert np.allclose(fd, g[f], rtol=1e-6, atol=1e-6 * np.linalg.norm(g[f])), (f, fd, g[f])
        assert np.all(abs_sum[f] >= np.abs(g[f]) - 1e-12)


def test_frames_at_one_pose_sum_to_the_single_pose_gradient():
    groups = _groups(_draws)
    T = _poses()[2]
    P = np.stack([T] * F)
    loss, g, _, _ = bo.evaluate(groups, P)
    tl, tg, tabs, _ = to.evaluate(groups, T)
    assert abs(loss - tl) <= 1e-12 * abs(tl)
    assert np.max(np.abs(g.sum(0) - tg)) <= 1e-12 * np.max(tabs)
    assert all(np.any(g[f] != 0) for f in range(F))


def test_a_ray_without_a_frame_contributes_nothing():
    """Rays whose draw has no frame (-1) leave the loss and every gradient: whatever their points and targets."""
    def frames(B, h):
        fr = _draws(B, h)
        fr[0, :3] = -1
        return fr
    a, b = _groups(frames), _groups(frames)
    bb = b[0]["batch"]
    bb["pcs"][0, :3] += 0.3
    bb["gt_depth"][0, :3] += 1.0
    bb["gt_colour"][0, :3] = 1.0 - bb["gt_colour"][0, :3]
    la, ga, _, _ = bo.evaluate(a, _poses())
    lb, gb, _, _ = bo.evaluate(b, _poses())
    assert abs(la - lb) <= 1e-13 * abs(la) and np.allclose(ga, gb, rtol=1e-12, atol=1e-15)
    lc, _, _, _ = bo.evaluate(_groups(_draws), _poses())
    assert lc != la


def test_window_update_closed_form():
    """Two iterations over a window of frames 0..3 with frame 0 held: per frame, Adam on its own tangent (the stacked
    Adam is element-wise); frame 3 has gradient 0 at iteration 2 and still moves by its momentum."""
    P0 = _poses()
    win = [0, 1, 2, 3]
    g1 = np.array([[9.0] * 6, [0.5, -2.0, 1e-3, 3.0, -0.25, 0.0], [1.0, 1.0, -1.0, 0.5, 0.5, -0.5],
                   [0.2, -0.3, 0.4, -0.5, 0.6, -0.7]])
    g2 = np.array([[9.0] * 6, [-0.5, 1.0, 2e-3, -1.0, 0.25, 1.0], [0.1, 0.2, 0.3, 0.4, 0.5, 0.6], [0.0] * 6])
    lr_r, lr_t = 1e-3, 2e-3
    P1, m, v = bo.window_update(P0, win, g1, None, None, 1, lr_r, lr_t, hold=0)
    P2, m2, v2 = bo.window_update(P1, win, g2, m, v, 2, lr_r, lr_t, hold=0)
    assert np.array_equal(P1[0], P0[0]) and np.array_equal(P2[0], P0[0])
    lr = np.array([lr_r] * 3 + [lr_t] * 3)
    for f in (1, 2, 3):
        d1 = -lr * g1[f] / (np.abs(g1[f]) + 1e-8)
        assert np.max(np.abs(P1[f, :3, :3] - to.exp_so3_np(d1[:3]) @ P0[f, :3, :3])) <= 1e-15
        assert np.max(np.abs(P1[f, :3, 3] - (P0[f, :3, 3] + d1[3:]))) <= 1e-15
        me = 0.9 * 0.1 * g1[f] + 0.1 * g2[f]
        ve = 0.999 * 0.001 * g1[f] ** 2 + 0.001 * g2[f] ** 2
        d2 = -lr * (me / (1 - 0.9 ** 2)) / (np.sqrt(ve / (1 - 0.999 ** 2)) + 1e-8)
        assert np.max(np.abs(P2[f, :3, :3] - to.exp_so3_np(d2[:3]) @ P1[f, :3, :3])) <= 1e-15
        assert np.max(np.abs(P2[f, :3, 3] - (P1[f, :3, 3] + d2[3:]))) <= 1e-15
    assert not np.array_equal(P2[3], P1[3])                 # zero gradient, moved by the momentum


def _fields(src, start, end):
    body = src[src.index(start):src.index(end)]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"[\s\*]([a-z_0-9]+)\s*(?:\[[A-Z_0-9]+\])?\s*[;,]", body)


def test_ba_structs_match_header_field_order():
    from vmap_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    for name, cls in (("vmb_ba_group", _lib.BaGroup), ("vmb_ba_target", _lib.BaTarget), ("vmb_ba_args", _lib.BaArgs),
                      ("vmb_sample_args", _lib.SampleArgs)):
        assert _fields(src, f"typedef struct {name}", f"}} {name};") == [f[0] for f in cls._fields_], name
    assert int(re.search(r"#define VMB_BA_MAX_WIN (\d+)", src).group(1)) == _lib.BA_MAX_WIN
    assert f"VMB_BA_ST_BAD_FRAME = {_lib.BA_ST_BAD_FRAME}" in src
    for n in ("vmb_ba_step", "vmb_ba_update"):
        assert n in _lib.EXPORTS and f"int {n}(" in src
