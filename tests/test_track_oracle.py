"""CPU checks of the tracking rule's restatement (oracle/track_oracle.py) and of the K10 binding."""
import math
import os
import re

import numpy as np
import torch

from oracle import track_oracle as to
from oracle import vmap_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _groups(seed=0):
    out = []
    for hidden, B, S, sc in ((32, 2, 10, 2.0), (64, 1, 14, 5.0)):
        params = vo.init_params(B, hidden, seed=seed + hidden, dtype=torch.float64)
        batch = vo.synthetic_batch(B, 12, S, seed=seed + hidden + 1, n_cam2surf=S - 9, dtype=torch.float64)
        out.append({"params": params, "scale": torch.full((B,), sc, dtype=torch.float64), "batch": batch})
    return out


def _pose():
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np([0.2, -0.1, 0.3])
    T[:3, 3] = [0.1, -0.2, 0.05]
    return T


def test_gradient_matches_central_differences():
    groups, T = _groups(), _pose()
    loss, g, abs_sum, _ = to.evaluate(groups, T)
    assert abs(loss - to.loss_at(groups, T)) <= 1e-12 * abs(loss)
    h = 1e-7
    fd = np.zeros(6)
    for i in range(6):
        e = np.zeros(6)
        e[i] = h
        fd[i] = (to.loss_at(groups, to.retract(T, e), var_pose=T) -
                 to.loss_at(groups, to.retract(T, -e), var_pose=T)) / (2 * h)
    # var is detached (loss.py:29), so the differences hold it at T; the L1 kinks make the loss piecewise smooth and
    # at a generic pose central differences then agree to O(h^2)
    assert np.allclose(fd, g, rtol=1e-6, atol=1e-6 * np.linalg.norm(g)), (fd, g)
    assert np.all(abs_sum >= np.abs(g) - 1e-12)


def test_per_object_empty_mask_rule():
    """A term whose own mask is empty is 0 for that object only (the reference would zero it for every object)."""
    groups = _groups()
    b = groups[0]["batch"]
    b["sem"][1] = 2
    b["mask_depth"][1] = False
    _, _, _, terms = to.evaluate(groups, _pose())
    t = terms[0]
    assert float(t[1, 0]) == 0.0 and float(t[1, 2]) == 0.0 and float(t[1, 1]) > 0.0
    assert float(t[0, 0]) > 0.0 and float(t[0, 2]) > 0.0


def test_exp_closed_form():
    th = 0.7
    Rz = np.array([[math.cos(th), -math.sin(th), 0], [math.sin(th), math.cos(th), 0], [0, 0, 1]])
    assert np.max(np.abs(to.exp_so3_np([0, 0, th]) - Rz)) <= 1e-15
    w = np.array([0.3, -0.4, 1.2])
    R = to.exp_so3_np(w)
    assert np.max(np.abs(R @ R.T - np.eye(3))) <= 1e-15 and abs(np.linalg.det(R) - 1) <= 1e-14
    assert np.max(np.abs(R @ w - w)) <= 1e-15                          # the axis is fixed
    tiny = np.array([1e-13, -2e-13, 5e-14])                            # below 1e-12: I + [w]x
    assert np.array_equal(to.exp_so3_np(tiny), np.eye(3) + to.hat(torch.from_numpy(tiny)).numpy())


def test_adam_closed_form():
    """Iteration 1: m^ = g, v^ = g^2, so delta = -lr g / (|g| + eps); iteration 2 from the stated recursions."""
    T0 = _pose()
    g1 = np.array([0.5, -2.0, 1e-3, 3.0, -0.25, 0.0])
    lr_r, lr_t = 1e-3, 2e-3
    T1, m, v = to.adam_update(T0, g1, None, None, 1, lr_r, lr_t)
    d = -np.array([lr_r] * 3 + [lr_t] * 3) * g1 / (np.abs(g1) + 1e-8)
    assert np.max(np.abs(T1[:3, :3] - to.exp_so3_np(d[:3]) @ T0[:3, :3])) <= 1e-15
    assert np.max(np.abs(T1[:3, 3] - (T0[:3, 3] + d[3:]))) <= 1e-15
    assert np.array_equal(T1[3], [0, 0, 0, 1])
    g2 = np.array([-0.5, 1.0, 2e-3, -1.0, 0.25, 1.0])
    T2, m2, v2 = to.adam_update(T1, g2, m, v, 2, lr_r, lr_t)
    me = 0.9 * 0.1 * g1 + 0.1 * g2
    ve = 0.999 * 0.001 * g1 * g1 + 0.001 * g2 * g2
    assert np.allclose(m2, me, rtol=1e-15, atol=0) and np.allclose(v2, ve, rtol=1e-15, atol=0)
    d2 = -np.array([lr_r] * 3 + [lr_t] * 3) * (me / (1 - 0.9 ** 2)) / (np.sqrt(ve / (1 - 0.999 ** 2)) + 1e-8)
    assert np.max(np.abs(T2[:3, 3] - (T1[:3, 3] + d2[3:]))) <= 1e-15


def _fields(src, start, end):
    body = src[src.index(start):src.index(end)]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"[\s\*]([a-z_0-9]+)\s*(?:\[[A-Z_0-9]+\])?\s*[;,]", body)


def test_track_structs_match_header_field_order():
    from vmap_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    assert _fields(src, "typedef struct vmb_track_group", "} vmb_track_group;") == \
        [f[0] for f in _lib.TrackGroup._fields_]
    assert _fields(src, "typedef struct vmb_track_args", "} vmb_track_args;") == [f[0] for f in _lib.TrackArgs._fields_]
    lim = dict(re.findall(r"#define (VMB_TRACK_[A-Z_]+) (\d+)", src))
    assert int(lim["VMB_TRACK_MAX_GROUPS"]) == _lib.TRACK_MAX_GROUPS and int(lim["VMB_TRACK_PART"]) == _lib.TRACK_PART
    assert f"VMB_TRACK_ST_BAD_ROW = {_lib.TRACK_ST_BAD_ROW}" in src
    for n in ("vmb_track_tiles", "vmb_track_step", "vmb_track_update"):
        assert n in _lib.EXPORTS and f"int {n}(" in src


def test_track_tiles_match_the_fp32_step_tiles():
    from vmap_b200 import _lib
    L = _lib.lib()
    for hidden, tp in ((32, 128), (64, 64), (128, 64), (256, 32)):
        for R, S in ((120, 10), (1200, 14), (7, 1)):
            assert L.vmb_track_tiles(hidden, R, S) == -(-R // (tp // S))
        assert L.vmb_track_tiles(hidden, 10, tp + 1) == -4


def _golden_groups():
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_track.npz"))
    out = {}
    for tag in ("obj", "bg"):
        params = {k: torch.from_numpy(g[f"{tag}_p_{k}"]) for k in vo.ALL_KEYS}
        batch = {k: torch.from_numpy(g[f"{tag}_in_{k}"]) for k in ("pcs", "z", "gt_depth", "gt_colour", "sem",
                                                                    "mask_depth")}
        B = batch["pcs"].shape[0]
        out[tag] = ({"params": params, "scale": torch.full((B,), float(g[f"{tag}_scale"]), dtype=torch.float64),
                     "batch": batch}, g[f"{tag}_pose"], float(g[f"{tag}_loss"]), g[f"{tag}_grad"])
    return out


def test_oracle_matches_reference_golden():
    """The restatement against the reference's own UniDirsEmbed / OccupancyMap / step_batch_loss, fp64 autograd."""
    for tag, (group, T, loss_ref, grad_ref) in _golden_groups().items():
        loss, g, _, _ = to.evaluate([group], T)
        assert abs(loss - loss_ref) <= 1e-10 * abs(loss_ref), tag
        assert np.max(np.abs(g - grad_ref)) <= 1e-10 * np.linalg.norm(grad_ref), (tag, g, grad_ref)


def test_loss_terms_equal_training_terms_when_masks_are_non_empty():
    """With every mask non-empty the per-object rule is the training loss (vmap_oracle.batch_loss_terms)."""
    for group in _groups():
        p, b = group["params"], group["batch"]
        alpha, colour = vo.forward(p, group["scale"], b["pcs"])
        mine = to.loss_terms(alpha, colour, b)
        ref = torch.stack(vo.batch_loss_terms(alpha, colour, b["gt_depth"], b["gt_colour"], b["sem"], b["mask_depth"],
                                              b["z"]), 1)
        assert torch.equal(mine, ref)
