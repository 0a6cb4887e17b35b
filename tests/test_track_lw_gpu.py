"""Tracking and bundle adjustment on the layer-wise tensor-core path (vmb_track_step_lw / vmb_ba_step_lw): parity with
K10 / K11 and the fp64 oracle, K10's partial-row layout, the BA rows, bitwise reproducibility, the fp16 clamp count,
the guards, localisation on a trained iMAP map and online SLAM in iMAP mode, and the vMAP background opt-in."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import track_lw_oracle as tlo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rand_pose(seed, rot_deg=20.0, trans=0.3):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    w *= math.radians(rot_deg) / np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w)
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _stack(hidden, B, R, S, seed, extra_rows=2):
    """A packed stack of B + extra_rows objects of which rows [1, 1 + B) are tracked, and a batch for them."""
    from vmap_b200.ensemble import VmapEnsemble
    n_rows = B + extra_rows
    params = vo.init_params(n_rows, hidden, seed=seed)
    ens = VmapEnsemble(n_rows, hidden=hidden, scale=2.0, impl="fp32")
    ens.load_stacked(params)
    rows = list(range(1, 1 + B))
    batch = vo.synthetic_batch(B, R, S, seed=seed + 1, n_cam2surf=S - 9 if S > 9 else 1)
    og = {"params": {k: v[rows] for k, v in params.items()}, "scale": torch.full((B,), 2.0), "batch": batch}
    return ens, rows, batch, og


def _track_once(ens, rows, batch, T, impl):
    """One iteration at zero rates: (per-object gradient [B, 6], per-object loss terms [B, 3], the partial rows, out)."""
    from vmap_b200.track import SampleGroup, track_samples
    sg = SampleGroup(ens, rows, batch, 1, impl=impl)
    sg.partials.fill_(float("nan"))
    out = track_samples([sg], T, 1, 0.0, 0.0)
    torch.cuda.synchronize()
    B = len(rows)
    part = sg.partials.view(B, -1, 10).cpu().numpy()
    return part[:, :, :6].sum(1), part[:, :, 6:9].sum(1), part, out


# Bars, about 4-5x the worst values an H100 (700 W) measured over the parity shapes and three seeds (the test prints
# them).  The per-object gradient error relative to the norm of that object's K10 gradient: worst 9.0e-2 (H 64, S 32;
# 1.3e-2 .. 3.8e-2 elsewhere) -- fp16 embedding, weights and activations on freshly initialised networks, whose pose
# gradients are small sums of large terms.  The loss terms' relative error: worst 1.2e-3.  The total gradient against
# the exact fp64 oracle, relative to its norm: worst 9.0e-2.  BA rows against K11 (summed error over sum |rows|): 2.0e-3.
LW_GRAD_BAR_K10, LW_TERM_BAR_K10 = 0.4, 5e-3
LW_GRAD_BAR_ORACLE = 0.4
LW_BA_BAR = 1e-2
# Against the fp16-faithful restatement (oracle/track_lw_oracle.py), which rounds where the path stores fp16: the
# per-object gradient error relative to the norm of the faithful gradient, the loss terms' relative error, and the BA
# rows' summed error over sum |rows|.  An H100 (700 W) measured worst 1.8e-2 (H 256, S 14; 4.3e-4 .. 3.4e-3 at every
# other shape), 4.5e-4 and 3.8e-4 (H 256, S 32); the bars are 4-5x those.
FAITHFUL_GRAD_BAR, FAITHFUL_TERM_BAR, FAITHFUL_BA_BAR = 8e-2, 2e-3, 2e-3


def _faithful(og, T, frames=None):
    return tlo.evaluate(og["params"], og["scale"], og["batch"], T, frames)


@pytest.mark.parametrize("hidden", [64, 128, 256])
@pytest.mark.parametrize("S,B,R", [(5, 1, 77), (10, 3, 61), (14, 2, 45), (32, 1, 33)])
def test_partials_parity_with_k10_and_oracle(hidden, S, B, R):
    worst = [0.0, 0.0, 0.0, 0.0, 0.0]
    for seed in (0, 1, 2):
        ens, rows, batch, og = _stack(hidden, B, R, S, seed=hidden + 7 * S + B + 100 * seed)
        T = _rand_pose(hidden + S + seed)
        g_lw, l_lw, part, out = _track_once(ens, rows, batch, T, "layerwise")
        g_k, l_k, part_k, _ = _track_once(ens, rows, batch, T, "fp32")
        # K10's partial-row count: vmb_track_tiles rows per object, every one written, nothing past them
        assert part.shape == part_k.shape and np.all(np.isfinite(part))
        assert int(out["status"][0]) & ~16 == 0, int(out["status"][0])
        for b in range(B):
            worst[0] = max(worst[0], np.abs(g_lw[b] - g_k[b]).max() / np.linalg.norm(g_k[b]))
            worst[1] = max(worst[1], (np.abs(l_lw[b] - l_k[b]) / np.maximum(np.abs(l_k[b]), 1e-12)).max())
        _, g, _, _ = to.evaluate([og], T)
        worst[2] = max(worst[2], np.abs(g_lw.sum(0) - g).max() / np.linalg.norm(g))
        f = _faithful(og, T)
        g_f, l_f = f["rows"].sum(1).numpy(), f["terms"][:, :3].numpy()
        for b in range(B):
            worst[3] = max(worst[3], np.abs(g_lw[b] - g_f[b]).max() / np.linalg.norm(g_f[b]))
            worst[4] = max(worst[4], (np.abs(l_lw[b] - l_f[b]) / np.maximum(np.abs(l_f[b]), 1e-12)).max())
    print(f"H{hidden} S{S} B{B} R{R}: grad vs K10 {worst[0]:.2e}, terms vs K10 {worst[1]:.2e}, grad vs oracle "
          f"{worst[2]:.2e}; vs faithful: grad {worst[3]:.2e}, terms {worst[4]:.2e}")
    assert worst[0] <= LW_GRAD_BAR_K10 and worst[1] <= LW_TERM_BAR_K10 and worst[2] <= LW_GRAD_BAR_ORACLE, worst
    assert worst[3] <= FAITHFUL_GRAD_BAR and worst[4] <= FAITHFUL_TERM_BAR, worst


def test_update_on_layerwise_partials_is_the_closed_form():
    """vmb_track_update, unchanged, on the new partials: one teacher-forced Adam / Exp step equals its fp64 closed form
    from the gradient the path produced."""
    from vmap_b200.track import SampleGroup, track_samples
    ens, rows, batch, _ = _stack(128, 2, 40, 14, seed=3)
    T = _rand_pose(5)
    sg = SampleGroup(ens, rows, batch, 1, impl="layerwise")
    out = track_samples([sg], T, 1, 1e-3, 2e-3)
    g = out["grad_hist"][0].cpu().numpy()
    # the update read the new partial rows: its gradient is their fp64 sum over objects and tiles
    gp = sg.partials.view(2, -1, 10)[..., :6].sum((0, 1)).cpu().numpy()
    assert np.abs(g - gp).max() <= 1e-12 * np.abs(gp).max()
    ref, _, _ = to.adam_update(T, g, np.zeros(6), np.zeros(6), 1, 1e-3, 2e-3)
    assert np.abs(out["pose"].cpu().numpy() - ref).max() <= 1e-12


def test_layerwise_is_bitwise_reproducible():
    ens, rows, batch, _ = _stack(256, 2, 50, 14, seed=4)
    T = _rand_pose(6)
    a = _track_once(ens, rows, batch, T, "layerwise")[2]
    b = _track_once(ens, rows, batch, T, "layerwise")[2]
    assert np.array_equal(a, b)


def _ba_once(ens, rows, batch, P, kf_draw, kf_frame, n_pix_draw, impl):
    from vmap_b200.ba import BaSampleGroup, ba_samples
    g = BaSampleGroup(ens, rows, batch, 1, n_pix_draw, kf_draw, kf_frame, impl=impl)
    out = ba_samples([g], P, list(range(1, P.shape[0])), 1, 0.0, 0.0)
    torch.cuda.synchronize()
    return g.ray_rows.view(len(rows), -1, 10).cpu().numpy(), out


@pytest.mark.parametrize("hidden,S", [(64, 10), (128, 14), (256, 32)])
def test_ba_rows_against_the_faithful_oracle(hidden, S):
    ens, rows, batch, og = _stack(hidden, 2, 60, S, seed=hidden + S)
    P = np.stack([np.eye(4), _rand_pose(1, 5, 0.05), _rand_pose(2, 5, 0.05)])
    kf_draw = np.array([[0, 1, 0, 1, 1, 0], [1, 1, 0, 0, 1, 0]], np.int32)    # 6 draws of 10 rays
    kf_frame = np.array([[1, 2], [2, 1]], np.int32)
    r_lw, out = _ba_once(ens, rows, batch, P, kf_draw, kf_frame, 10, "layerwise")
    frames = torch.from_numpy(np.stack([kf_frame[b][kf_draw[b]] for b in range(2)]).repeat(10, 1).astype(np.int64))
    r_f = _faithful(og, P, frames)["rows"].numpy()
    err = np.abs(r_lw[:, :, :6] - r_f).sum((0, 1)).max() / np.abs(r_f).sum()
    print(f"H{hidden} S{S}: BA rows vs faithful, summed error / sum |rows| {err:.2e}")
    assert err <= FAITHFUL_BA_BAR


def test_ba_rows_against_k11_and_the_track_flavour():
    ens, rows, batch, _ = _stack(128, 2, 60, 14, seed=8)
    P = np.stack([np.eye(4), _rand_pose(1, 5, 0.05), _rand_pose(2, 5, 0.05)])
    kf_draw = np.array([[0, 1, 0, 1, 1, 0]] * 2, np.int32)          # 6 draws of 10 rays
    kf_frame = np.array([[1, 2]] * 2, np.int32)
    r_lw, out = _ba_once(ens, rows, batch, P, kf_draw, kf_frame, 10, "layerwise")
    r_k, _ = _ba_once(ens, rows, batch, P, kf_draw, kf_frame, 10, "fp32")
    assert int(out["status"][0]) & ~16 == 0
    err = np.abs(r_lw[:, :, :6] - r_k[:, :, :6]).sum((0, 1)).max() / np.abs(r_k[:, :, :6]).sum()
    print(f"BA rows vs K11: summed gradient error / sum |rows| {err:.2e}")
    assert err <= LW_BA_BAR
    # every ray at one frame: the rows sum to the track flavour's partials (summation order aside)
    one = np.array([[1, 2]] * 2, np.int32)[:, :1].repeat(2, 1)
    r1, _ = _ba_once(ens, rows, batch, P, kf_draw, one, 10, "layerwise")
    g_t, l_t, _, _ = _track_once(ens, rows, batch, P[1], "layerwise")
    scale = np.abs(r1[:, :, :6]).sum()
    assert np.abs(r1[:, :, :6].sum(1) - g_t).max() <= 1e-12 * scale
    assert np.abs(r1[:, :, 6:9].sum(1) - l_t).max() <= 1e-12 * np.abs(l_t).sum()


def test_ba_bad_frame_and_empty_masks():
    ens, rows, batch, _ = _stack(64, 2, 40, 10, seed=9)
    P = np.stack([np.eye(4), _rand_pose(3, 5, 0.05)])
    kf_draw = np.array([[0, 1, 0, 1]] * 2, np.int32)
    kf_frame = np.array([[1, 7]] * 2, np.int32)                      # frame 7 is outside the table
    r, out = _ba_once(ens, rows, batch, P, kf_draw, kf_frame, 10, "layerwise")
    from vmap_b200 import _lib
    assert int(out["status"][0]) & _lib.BA_ST_BAD_FRAME
    bad = np.zeros(40, bool)
    bad[10:20] = bad[30:40] = True
    assert np.all(r[:, bad] == 0.0) and np.abs(r[:, ~bad, :6]).sum() > 0
    # object 1 has no valid depth ray: its depth term is 0 and the other object's terms are untouched
    b2 = {k: v.clone() for k, v in batch.items()}
    b2["mask_depth"][1] = False
    r2, _ = _ba_once(ens, rows, b2, P, kf_draw, np.array([[1, 1]] * 2, np.int32), 10, "layerwise")
    r0, _ = _ba_once(ens, rows, batch, P, kf_draw, np.array([[1, 1]] * 2, np.int32), 10, "layerwise")
    assert np.all(r2[1, :, 6] == 0.0) and np.array_equal(r2[0], r0[0])
    assert np.abs(r2[1, :, 7:9]).sum() > 0


def _saturating(params):
    """fused_oracle.saturation_batch alone stays far below the fp16 clamp at hidden 64 / 128 (the restatement's largest
    |2^8 dYc| is about 10 and |2^8 d_alpha w_a| about 1e3), so the out_color weights are raised: colour unit 0 is made a
    constant 2^-10 (a zero color_linear row, bias 2^-10), its out_color weights are set to 2^16, and the colour biases
    drop by the 2^6 that adds.  Its dYc column, 2^16 sum_c 2^8 dh_c, then passes 60000 at about a hundred points per
    object.  Its color_linear row is zero, so that column reaches no other gradient."""
    params["color_linear.0.weight"][:, 0] = 0.0
    params["color_linear.0.bias"][:, 0] = 2.0 ** -10
    params["out_color.weight"][:, :, 0] = 2.0 ** 16
    params["out_color.bias"] -= 2.0 ** 6
    return params


@pytest.mark.parametrize("hidden", [64, 128])
def test_clamp_count(hidden):
    """status[1]: the track and BA flavours count the same clamped values, between the restatement's counts of values
    clearly past and clearly within +-60000; an ordinary batch on the unmodified network counts none."""
    from oracle import fused_oracle as fo
    from vmap_b200 import _lib
    from vmap_b200.ensemble import VmapEnsemble
    B, R, S = 2, 64, 10
    rows = [1, 2]
    params = _saturating(vo.init_params(B + 2, hidden, seed=hidden))
    ens = VmapEnsemble(B + 2, hidden=hidden, scale=2.0, impl="fp32")
    ens.load_stacked(params)
    batch = fo.saturation_batch(B, R, S, seed=hidden + 1)
    T = _rand_pose(hidden, 5, 0.05)
    st = _track_once(ens, rows, batch, T, "layerwise")[3]["status"].cpu().numpy()
    assert st[0] & _lib.TRACK_ST_CLAMP and st[1] > 0, st
    # one draw of R rays per object, every ray at the frame whose pose is T
    _, out = _ba_once(ens, rows, batch, np.stack([np.eye(4), T]), np.zeros((B, 1), np.int32), np.ones((B, 1), np.int32),
                      R, "layerwise")
    assert int(out["status"][1]) == int(st[1])
    f = tlo.evaluate({k: v[rows] for k, v in params.items()}, torch.full((B,), 2.0), batch, T)
    lo = sum(int((f[k].abs() > 60000 * 1.05).sum()) for k in ("dyc_pre", "rank1"))
    hi = sum(int((f[k].abs() > 60000 / 1.05).sum()) for k in ("dyc_pre", "rank1"))
    print(f"H{hidden}: status[1] {int(st[1])}, restatement {lo} past 63000, {hi} past 57143")
    assert 0 < lo <= int(st[1]) <= hi
    ens0, rows0, batch0, _ = _stack(hidden, B, R, S, seed=hidden)
    st0 = _track_once(ens0, rows0, batch0, T, "layerwise")[3]["status"].cpu().numpy()
    assert st0[1] == 0 and not st0[0] & _lib.TRACK_ST_CLAMP, st0


def _bind_lw(ens, rows, batch, S_override=None):
    from vmap_b200 import _lib
    from vmap_b200.track import SampleGroup
    sg = SampleGroup(ens, rows, batch, 1)
    a = _lib.TrackArgs()
    a.n_groups, a.n_iter, a.iter = 1, 1, 1
    pose = torch.eye(4, dtype=torch.float64, device=DEV)
    status = torch.zeros(4, dtype=torch.int32, device=DEV)
    a.pose, a.status = C.c_void_p(pose.data_ptr()), C.c_void_p(status.data_ptr())
    a.colour_scaling, a.opacity_scaling = 5.0, 10.0
    sg.bind(a.group[0], 0)
    if S_override:
        a.group[0].n_samples = S_override
    keep = (sg, pose, status)
    return a, keep


def _call_lw(ens, a):
    return ens.lib.vmb_track_step_lw(ens._handle, C.byref(a), 0, C.c_void_p(ens.image.data_ptr()), None)


def test_guards():
    from vmap_b200 import _lib
    VMB_E_ARG, VMB_E_UNSUPPORTED = -1, -4
    ens32, rows, batch, _ = _stack(32, 1, 20, 10, seed=1)
    a, keep = _bind_lw(ens32, rows, batch)
    assert _call_lw(ens32, a) == VMB_E_UNSUPPORTED                   # hidden 32 stays on K10
    ens, rows, batch, _ = _stack(64, 2, 20, 10, seed=2)
    a, keep = _bind_lw(ens, rows, batch, S_override=33)
    assert _call_lw(ens, a) == VMB_E_UNSUPPORTED                     # S > 32
    a, keep = _bind_lw(ens, rows, batch)
    a.group[0].max_partials = 1
    assert _call_lw(ens, a) == VMB_E_ARG                             # partials too small
    a, keep = _bind_lw(ens, rows, batch)
    assert ens.lib.vmb_track_step_lw(ens._handle, C.byref(a), 0, None, None) == VMB_E_ARG   # no image
    # a row outside the stack: that object's rows are zero and the status bit is set; the other is unchanged
    a, (sg, pose, status) = _bind_lw(ens, rows, batch)
    assert _call_lw(ens, a) == 0
    torch.cuda.synchronize()
    good = sg.partials.clone()
    sg.rows_dev[1] = 99
    assert _call_lw(ens, a) == 0
    torch.cuda.synchronize()
    assert int(status[0]) & 4
    t = good.shape[0] // 2
    assert torch.all(sg.partials[t:] == 0) and torch.equal(sg.partials[:t], good[:t])


# ---- iMAP: localisation and online SLAM on the synthetic sphere room at 160 x 120 -----------------------------------
W, H, FX = 160, 120, 120.0
N = 24


def _imap_cfg():
    from vmap_b200.cfg import Config, replica_room0_dict
    d = replica_room0_dict(imap=True)
    d["camera"].update(w=W, h=H, fx=FX, fy=FX, cx=W / 2 - 0.5, cy=H / 2 - 0.5)
    return Config(config_dict=d)


@pytest.fixture(scope="module")
def seq():
    from vmap_b200 import synth
    return synth.sphere_room_sequence(N, W, H, FX, FX, W / 2 - 0.5, H / 2 - 0.5)


def _frame(seq, k):
    return (torch.from_numpy(seq["rgb"][k]), torch.from_numpy(seq["depth"][k].astype(np.float32)), None)


def _run(seq, n=N, poses=None, **kw):
    import random
    from vmap_b200.slam import Slam
    torch.manual_seed(0)
    random.seed(0)
    slam = Slam(_imap_cfg(), T_init=seq["poses"][0], **kw)
    for k in range(n):
        slam.step(*_frame(seq, k), T_wc=(poses if poses is not None else seq["poses"])[k])
    torch.cuda.synchronize()
    return slam


def _errors(T, G):
    dt = float(np.linalg.norm(T[:3, 3] - G[:3, 3]))
    c = np.clip((np.trace(T[:3, :3].T @ G[:3, :3]) - 1) / 2, -1, 1)
    return dt, math.degrees(math.acos(c))


@pytest.fixture(scope="module")
def imap_trained(seq):
    slam = _run(seq, track=False, seed=1)
    for _ in range(30):
        slam.loop.run()
    torch.cuda.synchronize()
    return slam


def _localise(slam, seq, k, T0, groups=None, n_iter=200, lr=3e-3):
    from vmap_b200.slam import tracker_groups
    from vmap_b200.track import Tracker, groups_from_objects
    store = slam.store
    rgb, depth, _ = _frame(seq, k)
    slot, _, _ = store.ingest(rgb, depth, torch.zeros(W, H, dtype=torch.int32), torch.from_numpy(T0))
    groups = groups or tracker_groups(groups_from_objects(slam.objects.values()), False, True)
    tr = Tracker(groups, slam.cfg, n_iter=n_iter, lr_rot=lr, lr_trans=lr, seed=k, impl="layerwise")
    pose, _ = tr.track(store, slot, T0, ids=[0])
    store.release(slot)
    return pose.cpu().numpy(), tr.status.cpu().numpy()


def _perturbations():
    from scipy.spatial.transform import Rotation
    out = []
    for ax in range(3):
        t = np.zeros(3); t[ax] = 0.10
        out.append((f"t{'xyz'[ax]}", np.eye(3), t))
    for ax in range(3):
        w = np.zeros(3); w[ax] = math.radians(5.0)
        out.append((f"r{'xyz'[ax]}", Rotation.from_rotvec(w).as_matrix(), np.zeros(3)))
    for j, (w, t) in enumerate([((1, -1, 1), (1, 1, -1)), ((-1, 1, 1), (1, -1, 1))]):
        w = np.array(w, float) / math.sqrt(3) * math.radians(5.0)
        t = np.array(t, float) / math.sqrt(3) * 0.10
        out.append((f"mix{j}", Rotation.from_rotvec(w).as_matrix(), t))
    return out


def _perturbed(G, R, t):
    T = G.copy()
    T[:3, :3] = G[:3, :3] @ R
    T[:3, 3] = G[:3, 3] + t
    return T


LOC_T_BAR, LOC_R_BAR = 0.02, 1.0      # test_slam_gpu.py's bars; an H100 (700 W) measured 0.15-0.57 cm / 0.05-0.06 deg


def test_imap_localisation_converges_on_a_trained_map(imap_trained, seq):
    worst, clamps = [0.0, 0.0], 0
    for k in (6, 17):
        G = seq["poses"][k]
        for name, R, t in _perturbations():
            pose, st = _localise(imap_trained, seq, k, _perturbed(G, R, t))
            dt, dr = _errors(pose, G)
            worst = [max(worst[0], dt), max(worst[1], dr)]
            clamps += int(st[1])
            assert int(st[0]) & 7 == 0, (k, name, st)
            assert dt <= LOC_T_BAR and dr <= LOC_R_BAR, (k, name, dt, dr)
    print(f"iMAP localisation, worst final error {worst[0] * 100:.3f} cm {worst[1]:.3f} deg; "
          f"fp16-clamped gradient values over the 16 runs: {clamps}")


def test_imap_localisation_on_a_fresh_map_misses_the_bars(imap_trained, seq):
    from vmap_b200 import synth
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.slam import tracker_groups
    from vmap_b200.track import groups_from_objects
    (ens, ids), = tracker_groups(groups_from_objects(imap_trained.objects.values()), False, True)
    fresh = VmapEnsemble(ens.n_obj, hidden=ens.hidden, scale=ens.scale.clone(), device=DEV)
    fresh.load_stacked(synth.init_params(ens.n_obj, ens.hidden, seed=9))
    met = 0
    G = seq["poses"][6]
    for name, R, t in _perturbations():
        pose, _ = _localise(imap_trained, seq, 6, _perturbed(G, R, t), groups=[(fresh, ids)])
        dt, dr = _errors(pose, G)
        met += dt <= LOC_T_BAR and dr <= LOC_R_BAR
    assert met == 0


# iMAP SLAM bar: an H100 (700 W) measured ATE rmse 1.98 / 3.59 / 4.18 cm over seeds 2/3/4 in one run and 2.98 / 1.92 /
# 2.77 and 2.17 / 2.69 / 4.05 cm in two more (3.10 / 2.09 / 2.47 cm with BA every 4 frames), and 3.46 cm with K10
# tracking (seed 2), so the spread is online mapping's, not the fp16 tracking path's; the mapping step's weight gradients sum with float atomics, so runs differ and the bar leaves room above the
# worst.  Holding every frame at T_0 (what Slam did in iMAP mode before id 0 was tracked) gives 12.5 cm, so the
# 4-5x rule of the parity bars cannot apply here: a bar of 4x the worst run (17 cm) would pass that control.  The bar
# sits between the runs and the control, at less than half the control.  K10 (impl "fp32") on the same sequence is
# printed as a reference for how much of the error is online mapping rather than the fp16 tracking path.
IMAP_ATE_BAR = 0.06


def test_imap_slam_end_to_end(seq):
    from vmap_b200 import metrics
    ates = []
    for seed in (2, 3, 4):
        res = _run(seq, track=True, graph=True, seed=seed).result()
        ate = metrics.ate(res["poses"], seq["poses"])["rmse"]
        ates.append(ate)
        assert not res["lost"].any() and all(t == [0] for t in res["tracked_ids"][1:])
        assert res["tracked_ids"][0] == [] and np.isfinite(res["track_loss"][1:]).all()
    # the control: what the code did before iMAP tracking, every frame mapped at T_0
    T0 = np.repeat(seq["poses"][:1], N, 0)
    ctrl = metrics.ate(np.repeat(seq["poses"][:1], N, 0), seq["poses"])["rmse"]
    ctrl_slam = _run(seq, track=False, poses=T0, seed=2).result()
    k10 = metrics.ate(_run(seq, track=True, graph=True, seed=2, track_impl="fp32").result()["poses"], seq["poses"])
    print(f"iMAP SLAM with K10 tracking (impl fp32), seed 2: ATE rmse {k10['rmse'] * 100:.3f} cm")
    assert np.array_equal(ctrl_slam["poses"], T0)
    print("iMAP SLAM ATE rmse (cm), seeds 2/3/4: " + ", ".join(f"{a * 100:.3f}" for a in ates) +
          f"; frames held at T_0: {ctrl * 100:.3f}")
    assert max(ates) < IMAP_ATE_BAR and ctrl > 2 * IMAP_ATE_BAR


def test_imap_slam_with_bundle_adjustment(seq):
    from vmap_b200 import metrics
    res = _run(seq, track=True, graph=True, seed=2, ba_every=4).result()
    ate = metrics.ate(res["poses"], seq["poses"])["rmse"]
    print(f"iMAP SLAM + BA every 4 frames: ATE rmse {ate * 100:.3f} cm; passes {sum(bool(f) for f in res['ba_frames'])}")
    assert not res["lost"].any() and ate < IMAP_ATE_BAR
    assert any(m == "replay" for m in res["ba_modes"])


def test_imap_tracker_graph_equals_eager(imap_trained, seq):
    """Tracker.capture / run replays the layer-wise frame bitwise equal to Tracker.track (a whole SLAM run is not
    bitwise reproducible in iMAP mode: the hidden-256 mapping step sums weight gradients with float atomics)."""
    from vmap_b200.slam import tracker_groups
    from vmap_b200.track import Tracker, groups_from_objects
    store = imap_trained.store
    rgb, depth, _ = _frame(seq, 9)
    T0 = _perturbed(seq["poses"][9], np.eye(3), np.array([0.03, -0.02, 0.01]))
    slot, _, _ = store.ingest(rgb, depth, torch.zeros(W, H, dtype=torch.int32), torch.from_numpy(T0))
    groups = tracker_groups(groups_from_objects(imap_trained.objects.values()), False, True)
    a = Tracker(groups, imap_trained.cfg, seed=3, impl="layerwise")
    b = Tracker(groups, imap_trained.cfg, seed=3, impl="layerwise")
    pa, la = a.track(store, slot, T0, ids=[0])
    b.capture(store, slot, T0, ids=[0])
    pb, lb = b.run(store, slot, T0)
    pc, lc = a.track(store, slot, T0, ids=[0])               # the second frame of `a`: the draw counter moved on
    pd, ld = b.run(store, slot, T0)
    torch.cuda.synchronize()
    store.release(slot)
    assert torch.equal(pa, pb) and torch.equal(la, lb) and torch.equal(pc, pd) and torch.equal(lc, ld)
    assert not torch.equal(pa, pc)


def test_imap_ba_replay_equals_eager(imap_trained):
    from vmap_b200.ba import BundleAdjuster
    from vmap_b200.track import groups_from_objects
    slam = imap_trained
    objs = dict(slam.objects)
    keep = slam.store.t_wc.clone()
    res = []
    for graph in (False, True):
        ba = BundleAdjuster(groups_from_objects(objs.values()), slam.cfg, objs, n_iter=5, seed=1, impl="layerwise")
        assert all(g.lw for g in ba.groups)
        poses = slam.poses.clone()
        for _ in range(2):
            if graph:
                ba.capture(slam.store, poses, objs)
                ba.replay(slam.store, poses, objs)
            else:
                ba.run(slam.store, poses, objs)
        torch.cuda.synchronize()
        res.append((poses.clone(), ba.losses.clone(), slam.store.t_wc.clone()))
        slam.store.t_wc.copy_(keep)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])
    assert not torch.equal(res[0][0], slam.poses)


def test_vmap_background_opt_in():
    """vMAP with do_bg: only the hidden-128 background group changes path; the run meets test_slam_gpu.py's bars."""
    import random
    from vmap_b200 import metrics, synth
    from vmap_b200.cfg import Config, replica_room0_dict
    from vmap_b200.slam import Slam
    s = synth.sphere_room_sequence(N, W, H, FX, FX, W / 2 - 0.5, H / 2 - 0.5)
    d = replica_room0_dict()
    d["camera"].update(w=W, h=H, fx=FX, fy=FX, cx=W / 2 - 0.5, cy=H / 2 - 0.5)
    torch.manual_seed(0)
    random.seed(0)
    slam = Slam(Config(config_dict=d), T_init=s["poses"][0], background_cls=s["background_cls"], seed=2,
                track_impl="layerwise")
    for k in range(N):
        slam.step(torch.from_numpy(s["rgb"][k]), torch.from_numpy(s["depth"][k].astype(np.float32)),
                  torch.from_numpy(s["inst"][k]), torch.from_numpy(s["cls"][k]))
    res = slam.result()
    lw = {g.ens.hidden: g.lw for g in slam.tracker.groups}
    assert lw == {32: False, 128: True}, lw
    ate, rpe = metrics.ate(res["poses"], s["poses"]), metrics.rpe(res["poses"], s["poses"])
    print(f"vMAP + layer-wise background: ATE rmse {ate['rmse'] * 100:.3f} cm, RPE {rpe['trans_rmse'] * 100:.3f} cm / "
          f"{rpe['rot_rmse_deg']:.3f} deg")
    assert not res["lost"].any()
    assert ate["rmse"] < 0.03 and rpe["trans_rmse"] < 0.015 and rpe["rot_rmse_deg"] < 0.8
