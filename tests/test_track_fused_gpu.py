"""Tracking and bundle adjustment of the hidden-32 objects on the fused wgmma tile (vmb_track_step_fused /
vmb_ba_step_fused): parity with the fp16-faithful restatement (oracle/track_fused_oracle.py, from the kernel's own
embedding), with K10 / K11 and with the fp64 oracle; K10's partial-row layout, the update on the new rows, the BA rows,
the weights the AdamW launch refreshed, bitwise reproducibility and graph replay, the guards, localisation on a
trained vMAP map and online vMAP SLAM."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import track_fused_oracle as tfo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo
from tests.test_fused_faithful_gpu import probe_embedding

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCALE = 2.0          # p / scale and eval_points' p * (1 / scale) agree bit for bit: the probe sees the kernel's points
SEEDS = (0, 1, 2)


def _rand_pose(seed, rot_deg=20.0, trans=0.3):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    w *= math.radians(rot_deg) / np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w)
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _stack(B, R, S, seed, extra_rows=2):
    """A packed hidden-32 stack of B + extra_rows objects of which rows [1, 1 + B) are tracked, and a batch for them."""
    from vmap_b200.ensemble import VmapEnsemble
    n_rows = B + extra_rows
    params = vo.init_params(n_rows, 32, seed=seed)
    ens = VmapEnsemble(n_rows, hidden=32, scale=SCALE, impl="fp32")
    ens.load_stacked(params)
    rows = list(range(1, 1 + B))
    batch = vo.synthetic_batch(B, R, S, seed=seed + 1, n_cam2surf=S - 9 if S > 9 else 1)
    og = {"params": {k: v[rows] for k, v in params.items()}, "scale": torch.full((B,), SCALE), "batch": batch}
    return ens, rows, batch, og


def _track_once(ens, rows, batch, T, impl, spare=16):
    """One iteration at zero rates: (per-object gradient [B, 6], per-object loss terms [B, 3], the partial rows
    [B, tiles, 10], out, the spare rows past them).  The partials buffer has ``spare`` NaN rows past the B * tiles the
    step may write."""
    from vmap_b200.track import SampleGroup, track_samples
    sg = SampleGroup(ens, rows, batch, 1, impl=impl)
    sg.partials = torch.full((len(rows) * sg.tiles + spare, 10), float("nan"), dtype=torch.float64, device=DEV)
    out = track_samples([sg], T, 1, 0.0, 0.0)
    torch.cuda.synchronize()
    B = len(rows)
    n = B * sg.tiles
    part = sg.partials[:n].view(B, -1, 10).cpu().numpy()
    return part[:, :, :6].sum(1), part[:, :, 6:9].sum(1), part, out, sg.partials[n:].cpu().numpy()


def _faithful(og, T, frames=None, kernel_emb=True):
    """The restatement, from the kernel's own embedding probed at the kernel's posed points."""
    emb = None
    if kernel_emb:
        t, _ = tfo.posed_points(T, frames, og["batch"]["pcs"].double(), SCALE)
        B, R, S, _ = t.shape
        pts = (t * SCALE).float().reshape(B, R * S, 3).to(DEV).contiguous()     # exact: SCALE is a power of two
        emb = probe_embedding(og["params"], SCALE, pts)
        emb = (emb[0].cpu(), emb[1].cpu())
    return tfo.evaluate(og["params"], og["scale"], og["batch"], T, frames, emb=emb)


def _rel(a, b):
    return np.abs(a - b).max() / max(np.linalg.norm(b), 1e-30)


def _term_rel(a, b):
    return (np.abs(a - b) / np.maximum(np.abs(b), 1e-12)).max()


# Bars, 4-5x the worst an H100 80GB HBM3 (700 W) measured over the shapes below and three seeds (the test prints them):
#   against the fp16-faithful restatement from the kernel's embedding: per-object gradient error relative to the norm
#   of the faithful gradient, worst 3.9e-4 (S 10, B 20, R 120); loss terms' relative error, worst 3.5e-4 (S 5, B 7);
#   against K10 (fp32 network): per-object gradient, worst 1.4e-1 (S 10, B 20: freshly initialised networks, whose
#   pose gradients are small sums of large terms, and the fp16 network); loss terms, worst 3.6e-3;
#   against the fp64 oracle: the group's gradient relative to its norm, worst 3.6e-2.
FAITHFUL_GRAD_BAR, FAITHFUL_TERM_BAR = 2e-3, 1.5e-3
K10_GRAD_BAR, K10_TERM_BAR = 0.6, 1.5e-2
ORACLE_GRAD_BAR = 0.15
# BA rows (summed error over sum |rows|): against the restatement, worst 2.7e-5 (S 10); against K11, worst 2.4e-3 (S 32)
FAITHFUL_BA_BAR, K11_BA_BAR = 1.2e-4, 1e-2

SHAPES = [(5, 1, 77), (5, 7, 50), (10, 3, 61), (10, 20, 120), (14, 2, 45), (14, 13, 37), (32, 1, 33), (32, 4, 20)]


@pytest.mark.parametrize("S,B,R", SHAPES, ids=["S{}B{}R{}".format(*c) for c in SHAPES])
def test_partials_parity(S, B, R):
    from vmap_b200 import _lib
    worst = [0.0] * 5
    for seed in SEEDS:
        ens, rows, batch, og = _stack(B, R, S, seed=7 * S + B + 100 * seed)
        T = _rand_pose(S + B + seed)
        g_f, l_f, part, out, spare = _track_once(ens, rows, batch, T, "fused")
        g_k, l_k, part_k, _, _ = _track_once(ens, rows, batch, T, "fp32")
        # K10's partial-row count: vmb_track_tiles rows per object, every one written, nothing past them
        assert part.shape[1] == ens.lib.vmb_track_tiles(32, R, S) and part.shape == part_k.shape
        assert np.all(np.isfinite(part)) and np.all(np.isnan(spare)) and np.all(part[:, :, 9] == 0)
        assert int(out["status"][0]) & ~_lib.TRACK_ST_CLAMP == 0, int(out["status"][0])
        f = _faithful(og, T)
        gf, lf = f["rows"].sum(1).numpy(), f["terms"][:, :3].numpy()
        for b in range(B):
            worst[0] = max(worst[0], _rel(g_f[b], gf[b]))
            worst[1] = max(worst[1], _term_rel(l_f[b], lf[b]))
            worst[2] = max(worst[2], _rel(g_f[b], g_k[b]))
            worst[3] = max(worst[3], _term_rel(l_f[b], l_k[b]))
        _, g, _, _ = to.evaluate([og], T)
        worst[4] = max(worst[4], _rel(g_f.sum(0), g))
    print(f"S{S} B{B} R{R}: vs faithful grad {worst[0]:.2e} (bar {FAITHFUL_GRAD_BAR:.0e}), terms {worst[1]:.2e} "
          f"(bar {FAITHFUL_TERM_BAR:.0e}); vs K10 grad {worst[2]:.2e} (bar {K10_GRAD_BAR:.0e}), terms {worst[3]:.2e} "
          f"(bar {K10_TERM_BAR:.0e}); vs fp64 oracle {worst[4]:.2e} (bar {ORACLE_GRAD_BAR:.0e})")
    assert worst[0] <= FAITHFUL_GRAD_BAR and worst[1] <= FAITHFUL_TERM_BAR, worst
    assert worst[2] <= K10_GRAD_BAR and worst[3] <= K10_TERM_BAR and worst[4] <= ORACLE_GRAD_BAR, worst


def test_update_on_fused_partials_is_the_closed_form():
    """vmb_track_update, unchanged, on the new partials: one Adam / Exp step equals its fp64 closed form from the
    gradient the path produced."""
    from vmap_b200.track import SampleGroup, track_samples
    ens, rows, batch, _ = _stack(3, 40, 14, seed=3)
    T = _rand_pose(5)
    sg = SampleGroup(ens, rows, batch, 1, impl="fused")
    assert sg.path == "fused"
    out = track_samples([sg], T, 1, 1e-3, 2e-3)
    g = out["grad_hist"][0].cpu().numpy()
    gp = sg.partials.view(3, -1, 10)[..., :6].sum((0, 1)).cpu().numpy()
    assert np.abs(g - gp).max() <= 1e-12 * np.abs(gp).max()
    ref, _, _ = to.adam_update(T, g, np.zeros(6), np.zeros(6), 1, 1e-3, 2e-3)
    assert np.abs(out["pose"].cpu().numpy() - ref).max() <= 1e-12


def test_fused_is_bitwise_reproducible():
    ens, rows, batch, _ = _stack(6, 50, 14, seed=4)
    T = _rand_pose(6)
    a = _track_once(ens, rows, batch, T, "fused")[2]
    b = _track_once(ens, rows, batch, T, "fused")[2]
    assert np.array_equal(a, b)


def _ba_once(ens, rows, batch, P, kf_draw, kf_frame, n_pix_draw, impl):
    from vmap_b200.ba import BaSampleGroup, ba_samples
    g = BaSampleGroup(ens, rows, batch, 1, n_pix_draw, kf_draw, kf_frame, impl=impl)
    out = ba_samples([g], P, list(range(1, P.shape[0])), 1, 0.0, 0.0)
    torch.cuda.synchronize()
    return g.ray_rows.view(len(rows), -1, 10).cpu().numpy(), out


@pytest.mark.parametrize("S", [5, 10, 14, 32])
def test_ba_rows_against_k11_and_the_restatement(S):
    from vmap_b200 import _lib
    worst = [0.0, 0.0]
    for seed in SEEDS:
        ens, rows, batch, og = _stack(2, 60, S, seed=S + 10 * seed)
        P = np.stack([np.eye(4), _rand_pose(1 + seed, 5, 0.05), _rand_pose(2 + seed, 5, 0.05)])
        kf_draw = np.array([[0, 1, 0, 1, 1, 0], [1, 1, 0, 0, 1, 0]], np.int32)    # 6 draws of 10 rays
        kf_frame = np.array([[1, 2], [2, 1]], np.int32)
        r_f, out = _ba_once(ens, rows, batch, P, kf_draw, kf_frame, 10, "fused")
        r_k, _ = _ba_once(ens, rows, batch, P, kf_draw, kf_frame, 10, "fp32")
        assert int(out["status"][0]) & ~_lib.TRACK_ST_CLAMP == 0 and np.all(r_f[:, :, 9] == 0)
        frames = torch.from_numpy(np.stack([kf_frame[b][kf_draw[b]] for b in range(2)]).repeat(10, 1).astype(np.int64))
        r_o = _faithful(og, P, frames)["rows"].numpy()
        worst[0] = max(worst[0], np.abs(r_f[:, :, :6] - r_o).sum((0, 1)).max() / np.abs(r_o).sum())
        worst[1] = max(worst[1], np.abs(r_f[:, :, :6] - r_k[:, :, :6]).sum((0, 1)).max() / np.abs(r_k[:, :, :6]).sum())
    print(f"S{S}: BA rows, summed error / sum |rows|: vs faithful {worst[0]:.2e} (bar {FAITHFUL_BA_BAR:.0e}), vs K11 "
          f"{worst[1]:.2e} (bar {K11_BA_BAR:.0e})")
    assert worst[0] <= FAITHFUL_BA_BAR and worst[1] <= K11_BA_BAR, worst


@pytest.mark.parametrize("S", [5, 10, 14])
def test_ba_rows_at_one_frame_are_the_track_flavour(S):
    ens, rows, batch, _ = _stack(3, 60, S, seed=8 + S)
    P = np.stack([np.eye(4), _rand_pose(1, 5, 0.05), _rand_pose(2, 5, 0.05)])
    kf_draw = np.array([[0, 1, 0, 1, 1, 0]] * 3, np.int32)
    one = np.array([[1, 1]] * 3, np.int32)
    r1, _ = _ba_once(ens, rows, batch, P, kf_draw, one, 10, "fused")
    g_t, l_t, part, _, _ = _track_once(ens, rows, batch, P[1], "fused")
    # the track flavour's tiles are the BA rows summed in ray order: the same per-ray values, only the grouping differs
    scale = np.abs(r1[:, :, :6]).sum()
    assert np.abs(r1[:, :, :6].sum(1) - g_t).max() <= 1e-12 * scale
    assert np.abs(r1[:, :, 6:9].sum(1) - l_t).max() <= 1e-12 * np.abs(l_t).sum()
    nr10 = 128 // S
    for j in range(part.shape[1]):
        acc = np.zeros((3, 9))
        for r in range(j * nr10, min(60, (j + 1) * nr10)):
            acc += r1[:, r, :9]
        assert np.array_equal(part[:, j, :9], acc), j


def test_ba_bad_frame_bad_row_and_empty_masks():
    from vmap_b200 import _lib
    ens, rows, batch, _ = _stack(3, 40, 10, seed=9)
    P = np.stack([np.eye(4), _rand_pose(3, 5, 0.05)])
    kf_draw = np.array([[0, 1, 0, 1]] * 3, np.int32)
    kf_frame = np.array([[1, 7]] * 3, np.int32)                      # frame 7 is outside the table
    r, out = _ba_once(ens, rows, batch, P, kf_draw, kf_frame, 10, "fused")
    assert int(out["status"][0]) & _lib.BA_ST_BAD_FRAME
    bad = np.zeros(40, bool)
    bad[10:20] = bad[30:40] = True
    assert np.all(r[:, bad] == 0.0) and np.abs(r[:, ~bad, :6]).sum() > 0
    # object 1 has no valid depth ray: only its depth term is 0, the other objects' rows are unchanged
    ok = np.array([[1, 1]] * 3, np.int32)
    r0, _ = _ba_once(ens, rows, batch, P, kf_draw, ok, 10, "fused")
    b2 = {k: v.clone() for k, v in batch.items()}
    b2["mask_depth"][1] = False
    r2, _ = _ba_once(ens, rows, b2, P, kf_draw, ok, 10, "fused")
    assert np.all(r2[1, :, 6] == 0.0) and np.abs(r2[1, :, 7:9]).sum() > 0 and np.abs(r0[1, :, 6]).sum() > 0
    assert np.array_equal(r2[0], r0[0]) and np.array_equal(r2[2], r0[2])
    # a row outside the stack: that object's rows are zero and the status bit is set; the others are unchanged
    from vmap_b200.ba import BaSampleGroup, ba_samples
    g = BaSampleGroup(ens, rows, batch, 1, 10, kf_draw, ok, impl="fused")
    g.rows_dev[1] = 99
    out = ba_samples([g], P, [1], 1, 0.0, 0.0)
    torch.cuda.synchronize()
    r3 = g.ray_rows.view(3, -1, 10).cpu().numpy()
    assert int(out["status"][0]) & _lib.TRACK_ST_BAD_ROW
    assert np.all(r3[1] == 0.0) and np.array_equal(r3[0], r0[0]) and np.array_equal(r3[2], r0[2])


def test_reads_the_image_the_adamw_launch_refreshed():
    """After a few mapping steps (AdamW rewrote params and the fp16 image), the step reads the new weights: its rows
    match K10 on the updated params within the parity bars, and differ from the rows before the steps."""
    ens, rows, batch, og = _stack(4, 60, 10, seed=11, extra_rows=1)
    T = _rand_pose(12)
    g0 = _track_once(ens, rows, batch, T, "fused")[0]
    mb = vo.synthetic_batch(ens.n_obj, 256, 10, seed=13, n_cam2surf=1)
    p0 = ens.params.clone()
    for _ in range(5):
        ens.forward_backward({k: v.to(DEV) for k, v in mb.items()})
        ens.adam_step()
    torch.cuda.synchronize()
    assert (ens.params - p0).abs().max() > 1e-3
    g_f, l_f = _track_once(ens, rows, batch, T, "fused")[:2]
    g_k, l_k = _track_once(ens, rows, batch, T, "fp32")[:2]
    err = max(_rel(g_f[b], g_k[b]) for b in range(4))
    moved = min(_rel(g_f[b], g0[b]) for b in range(4))
    print(f"after 5 mapping steps: vs K10 on the new params {err:.2e}; moved from the old rows by {moved:.2e}")
    assert err <= K10_GRAD_BAR and max(_term_rel(l_f[b], l_k[b]) for b in range(4)) <= K10_TERM_BAR
    assert moved > 10 * err


# ---- the guards -------------------------------------------------------------------------------------------------------

def _bind(ens, rows, batch, S_override=None):
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
    return a, (sg, pose, status)


def _call(ens, a, image=True):
    return ens.lib.vmb_track_step_fused(ens._handle, C.byref(a), 0, C.c_void_p(ens.image.data_ptr()) if image else None,
                                        None)


def test_guards():
    from vmap_b200 import _lib
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.track import SampleGroup
    VMB_E_ARG, VMB_E_UNSUPPORTED = -1, -4
    ens64 = VmapEnsemble(3, hidden=64, scale=SCALE, impl="fp32")
    ens64.load_stacked(vo.init_params(3, 64, seed=1))
    b64 = vo.synthetic_batch(2, 20, 10, seed=2, n_cam2surf=1)
    a, keep = _bind(ens64, [1, 2], b64)
    assert _call(ens64, a) == VMB_E_UNSUPPORTED                      # hidden 64 takes the layer-wise pair
    ens, rows, batch, _ = _stack(2, 20, 10, seed=2)
    a, keep = _bind(ens, rows, batch, S_override=33)
    assert _call(ens, a) == VMB_E_UNSUPPORTED                        # S > 32
    a, keep = _bind(ens, rows, batch)
    a.group[0].max_partials = 1
    assert _call(ens, a) == VMB_E_ARG                                # partials too small
    a, keep = _bind(ens, rows, batch)
    assert _call(ens, a, image=False) == VMB_E_ARG                   # no image
    # a row outside the stack: that object's partials are zero and the status bit is set; the other is unchanged
    a, (sg, pose, status) = _bind(ens, rows, batch)
    assert _call(ens, a) == 0
    torch.cuda.synchronize()
    good = sg.partials.clone()
    sg.rows_dev[1] = 99
    assert _call(ens, a) == 0
    torch.cuda.synchronize()
    assert int(status[0]) & _lib.TRACK_ST_BAD_ROW
    t = good.shape[0] // 2
    assert torch.all(sg.partials[t:] == 0) and torch.equal(sg.partials[:t], good[:t])
    # a hidden-32 group without its fp16 image does not fall back to K10
    ens.image = None
    with pytest.raises(_lib.VmbError):
        SampleGroup(ens, rows, batch, 1, impl="fused")
    assert SampleGroup(ens, rows, batch, 1, impl="layerwise").path == "fp32"


# ---- localisation on a trained vMAP map and online vMAP SLAM: the sphere room of test_slam_gpu.py ------------------
from tests.test_slam_gpu import (LOC_R_BAR, LOC_T_BAR, SLAM_ATE_BAR, SLAM_RPE_R_BAR, SLAM_RPE_T_BAR,  # noqa: E402
                                 _errors, _frame, _map_groups, _perturbations, _perturbed, _run, seq, trained)  # noqa: E402,F401


def _localise(slam, seq, k, T0, groups=None, n_iter=200, lr=3e-3):
    from vmap_b200.track import Tracker
    store = slam.store
    rgb, depth, inst, cls = _frame(seq, k)
    slot, _, _ = store.ingest(rgb, depth, inst, torch.from_numpy(T0), cls=cls, background_cls=seq["background_cls"])
    groups = groups or _map_groups(slam)
    ids = [i for i in store.visible_objects() if i != 0]
    tr = Tracker(groups, slam.cfg, n_iter=n_iter, lr_rot=lr, lr_trans=lr, seed=k, impl="fused")
    assert all(g.path == "fused" for g in tr.groups)
    pose, _ = tr.track(store, slot, T0, ids=ids)
    store.release(slot)
    return pose.cpu().numpy(), tr.status.cpu().numpy()


def test_localisation_converges_on_a_trained_map(trained, seq):
    worst, clamps = [0.0, 0.0], 0
    for k in (6, 17):
        G = seq["poses"][k]
        for name, R, t in _perturbations():
            pose, st = _localise(trained, seq, k, _perturbed(G, R, t))
            dt, dr = _errors(pose, G)
            worst = [max(worst[0], dt), max(worst[1], dr)]
            clamps += int(st[1])
            assert int(st[0]) & 7 == 0, (k, name, st)
            assert dt <= LOC_T_BAR and dr <= LOC_R_BAR, (k, name, dt, dr)
    print(f"vMAP localisation on the fused path, worst final error {worst[0] * 100:.3f} cm {worst[1]:.3f} deg "
          f"(bars {LOC_T_BAR * 100:.0f} cm, {LOC_R_BAR:.0f} deg); fp16-clamped head gradients over the 16 runs: {clamps}")


def test_localisation_on_a_fresh_map_misses_the_bars(trained, seq):
    from vmap_b200 import synth
    from vmap_b200.ensemble import VmapEnsemble
    (ens, ids), = _map_groups(trained)
    fresh = VmapEnsemble(ens.n_obj, hidden=ens.hidden, scale=ens.scale.clone(), device=DEV)
    fresh.load_stacked(synth.init_params(ens.n_obj, ens.hidden, seed=9))
    met = 0
    G = seq["poses"][6]
    for name, R, t in _perturbations():
        pose, _ = _localise(trained, seq, 6, _perturbed(G, R, t), groups=[(fresh, ids)])
        dt, dr = _errors(pose, G)
        met += dt <= LOC_T_BAR and dr <= LOC_R_BAR
    assert met == 0


def test_tracked_set_grows_after_a_capture(trained, seq):
    """An object back in view: after a capture with k objects, a frame that tracks k + 1 on the same ensemble runs
    (the track flavour's workspace is sized for the handle, not for the frame's tracked set) and equals a tracker that
    never captured.  A copy of the trained stack gives a handle no earlier test has grown."""
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.track import Tracker
    (ens, names), = _map_groups(trained)
    copy = VmapEnsemble(ens.n_obj, hidden=ens.hidden, scale=ens.scale.clone(), device=DEV)
    copy.load_stacked(ens.stacked())
    store = trained.store
    rgb, depth, inst, cls = _frame(seq, 9)
    T0 = _perturbed(seq["poses"][9], np.eye(3), np.array([0.03, -0.02, 0.01]))
    slot, _, _ = store.ingest(rgb, depth, inst, torch.from_numpy(T0), cls=cls, background_cls=seq["background_cls"])
    ids = sorted(i for i in store.visible_objects() if i != 0)
    assert len(ids) >= 2, ids
    few = ids[:-1]
    a = Tracker([(copy, names)], trained.cfg, seed=5, impl="fused")
    b = Tracker([(copy, names)], trained.cfg, seed=5, impl="fused")
    a.track(store, slot, T0, ids=few)
    a.capture(store, slot, T0, ids=few)
    pa1, la1 = a.run(store, slot, T0)
    b.track(store, slot, T0, ids=few)
    pb1, lb1 = b.track(store, slot, T0, ids=few)
    pa2, la2 = a.track(store, slot, T0, ids=ids)              # k + 1 objects, eagerly, after the capture
    pb2, lb2 = b.track(store, slot, T0, ids=ids)
    a.capture(store, slot, T0, ids=ids)                       # and the larger set captures and replays too
    pa3, la3 = a.run(store, slot, T0)
    pb3, lb3 = b.track(store, slot, T0, ids=ids)
    torch.cuda.synchronize()
    store.release(slot)
    assert len(a.groups[0].active) == len(few) + 1 and int(a.status[0]) & 7 == 0 and int(b.status[0]) & 7 == 0
    assert torch.equal(pa1, pb1) and torch.equal(la1, lb1) and torch.equal(pa2, pb2) and torch.equal(la2, lb2)
    assert torch.equal(pa3, pb3) and torch.equal(la3, lb3) and torch.isfinite(la2).all()


def test_tracker_graph_equals_eager(trained, seq):
    from vmap_b200.track import Tracker
    store = trained.store
    rgb, depth, inst, cls = _frame(seq, 9)
    T0 = _perturbed(seq["poses"][9], np.eye(3), np.array([0.03, -0.02, 0.01]))
    slot, _, _ = store.ingest(rgb, depth, inst, torch.from_numpy(T0), cls=cls, background_cls=seq["background_cls"])
    ids = [i for i in store.visible_objects() if i != 0]
    a = Tracker(_map_groups(trained), trained.cfg, seed=3, impl="fused")
    b = Tracker(_map_groups(trained), trained.cfg, seed=3, impl="fused")
    pa, la = a.track(store, slot, T0, ids=ids)
    b.capture(store, slot, T0, ids=ids)
    pb, lb = b.run(store, slot, T0)
    pc, lc = a.track(store, slot, T0, ids=ids)               # the second frame of `a`: the draw counter moved on
    pd, ld = b.run(store, slot, T0)
    torch.cuda.synchronize()
    store.release(slot)
    assert torch.equal(pa, pb) and torch.equal(la, lb) and torch.equal(pc, pd) and torch.equal(lc, ld)
    assert not torch.equal(pa, pc)


def test_ba_replay_equals_eager(trained):
    from vmap_b200.ba import BundleAdjuster
    from vmap_b200.track import groups_from_objects
    slam = trained
    objs = dict(slam.objects)
    keep = slam.store.t_wc.clone()
    res = []
    for graph in (False, True):
        ba = BundleAdjuster(groups_from_objects(objs.values()), slam.cfg, objs, n_iter=5, seed=1, impl="fused")
        assert all(g.path == "fused" for g in ba.groups)
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


def _slam(seq, do_bg, **kw):
    from vmap_b200 import metrics
    from tests.test_slam_gpu import _cfg
    slam = _run(seq, track=True, graph=True, seed=2, cfg=_cfg(do_bg), track_impl="fused", **kw)
    res = slam.result()
    paths = {g.ens.hidden: g.path for g in slam.tracker.groups}
    ate, rpe = metrics.ate(res["poses"], seq["poses"]), metrics.rpe(res["poses"], seq["poses"])
    return slam, res, paths, ate, rpe


@pytest.mark.parametrize("do_bg", [False, True])
def test_vmap_slam_on_the_fused_path(seq, do_bg):
    slam, res, paths, ate, rpe = _slam(seq, do_bg)
    print(f"vMAP SLAM, fused tracking, do_bg {int(do_bg)}: ATE rmse {ate['rmse'] * 100:.3f} cm, RPE "
          f"{rpe['trans_rmse'] * 100:.3f} cm / {rpe['rot_rmse_deg']:.3f} deg (bars {SLAM_ATE_BAR * 100:.1f} cm, "
          f"{SLAM_RPE_T_BAR * 100:.1f} cm / {SLAM_RPE_R_BAR:.1f} deg)")
    assert paths == ({32: "fused", 128: "layerwise"} if do_bg else {32: "fused"}), paths
    assert not res["lost"].any() and np.all(np.isfinite(res["track_loss"][1:]))
    assert "replay" in res["track_modes"]
    assert ate["rmse"] < SLAM_ATE_BAR and rpe["trans_rmse"] < SLAM_RPE_T_BAR and rpe["rot_rmse_deg"] < SLAM_RPE_R_BAR


def test_vmap_slam_with_fused_bundle_adjustment(seq):
    slam, res, paths, ate, rpe = _slam(seq, False, ba_every=4, ba_impl="fused")
    print(f"vMAP SLAM, fused tracking + fused BA every 4 frames: ATE rmse {ate['rmse'] * 100:.3f} cm, RPE "
          f"{rpe['trans_rmse'] * 100:.3f} cm / {rpe['rot_rmse_deg']:.3f} deg; passes "
          f"{sum(bool(f) for f in res['ba_frames'])}")
    assert all(g.path == "fused" for g in slam.ba.groups)
    assert not res["lost"].any() and any(m == "replay" for m in res["ba_modes"])
    assert ate["rmse"] < SLAM_ATE_BAR and rpe["trans_rmse"] < SLAM_RPE_T_BAR and rpe["rot_rmse_deg"] < SLAM_RPE_R_BAR
