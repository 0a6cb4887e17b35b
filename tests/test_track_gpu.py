"""K10 camera tracking on the GPU: gradient parity with the fp64 oracle, the teacher-forced Adam / Exp loop, the
per-object empty-mask rule, bitwise reproducibility (two runs, eager against graph replay) and argument checks."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import track_oracle as to
from oracle import vmap_oracle as vo

pytestmark = pytest.mark.gpu


def _rand_pose(seed, rot_deg=20.0, trans=0.3):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    w *= math.radians(rot_deg) / np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w)
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _group(hidden, B, R, S, seed, extra_rows=2, n_iter=1):
    """A packed stack of B + extra_rows objects of which rows [1, 1+B) are tracked (a strided subset)."""
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.track import SampleGroup
    n_rows = B + extra_rows
    params = vo.init_params(n_rows, hidden, seed=seed)
    ens = VmapEnsemble(n_rows, hidden=hidden, scale=2.0, impl="fp32")
    ens.load_stacked(params)
    r0 = min(1, extra_rows)
    rows = list(range(r0, r0 + B))
    batch = vo.synthetic_batch(B, R * n_iter, S, seed=seed + 1, n_cam2surf=S - 9)
    sg = SampleGroup(ens, rows, batch, n_iter)
    og = {"params": {k: v[rows] for k, v in params.items()}, "scale": torch.full((B,), 2.0), "batch": batch}
    return sg, og


def _check_grad(gk, go, abs_sum):
    tol = 1e-4 * np.linalg.norm(go) + 1e-4 * abs_sum
    assert np.all(np.abs(gk - go) <= tol), (gk, go, tol)


def _check_terms(tk, to_):
    assert np.all(np.abs(tk - to_) <= 1e-5 * np.abs(to_) + 1e-7), (tk, to_)


@pytest.mark.parametrize("hidden", [32, 64, 128, 256])
@pytest.mark.parametrize("S", [10, 14])
@pytest.mark.parametrize("B", [1, 3, 20])
def test_gradient_parity(hidden, S, B):
    from vmap_b200.track import track_samples
    R = 24 if B == 20 else 40
    sg, og = _group(hidden, B, R, S, seed=hidden * 7 + S * 3 + B)
    T = _rand_pose(hidden + S + B)
    out = track_samples([sg], T, 1, 0.0, 0.0)
    loss, g, abs_sum, terms = to.evaluate([og], T)
    _check_grad(out["grad_hist"][0].cpu().numpy(), g, abs_sum)
    _check_terms(sg.loss_terms.double().cpu().numpy(), terms[0].numpy())
    assert abs(float(out["losses"][0]) - loss) <= 1e-5 * abs(loss)
    assert np.array_equal(out["pose"].cpu().numpy(), T)          # zero rates leave the pose as it was
    assert int(out["status"][0]) == 0


def test_two_groups_sum():
    """An object stack and a background model in one problem: the update sums both groups."""
    from vmap_b200.track import track_samples
    s1, o1 = _group(32, 3, 30, 10, seed=5)
    s2, o2 = _group(128, 1, 60, 14, seed=6, extra_rows=0)
    T = _rand_pose(11)
    out = track_samples([s1, s2], T, 1, 0.0, 0.0)
    loss, g, abs_sum, terms = to.evaluate([o1, o2], T)
    _check_grad(out["grad_hist"][0].cpu().numpy(), g, abs_sum)
    _check_terms(s2.loss_terms.double().cpu().numpy(), terms[1].numpy())
    assert abs(float(out["losses"][0]) - loss) <= 1e-5 * abs(loss)


def test_teacher_forced_loop():
    """Each iteration's kernel gradient matches the oracle at the kernel's own pose; each pose update is the fp64
    closed form applied to the kernel's own gradient."""
    from vmap_b200.track import track_samples
    n_iter, R = 10, 30
    sg, og = _group(32, 3, R, 10, seed=21, n_iter=n_iter)
    T0 = _rand_pose(3, rot_deg=5.0, trans=0.1)
    lr_rot, lr_trans = 2e-3, 1e-3
    out = track_samples([sg], T0, n_iter, lr_rot, lr_trans)
    poses = out["pose_hist"].cpu().numpy()
    grads = out["grad_hist"].cpu().numpy()
    assert np.array_equal(poses[0], T0)
    m = v = np.zeros(6)
    for i in range(n_iter):
        sl = to.slice_groups([og], i, [R])
        _, g, abs_sum, _ = to.evaluate(sl, poses[i])
        _check_grad(grads[i], g, abs_sum)
        T1, m, v = to.adam_update(poses[i], grads[i], m, v, i + 1, lr_rot, lr_trans)
        assert np.max(np.abs(T1 - poses[i + 1])) <= 1e-12, i
    assert not np.array_equal(poses[-1], poses[0])


def test_per_object_empty_mask():
    """An object whose rays are all unknown with no valid depth has empty depth and opacity masks: those terms are 0
    for it alone, and the other objects' terms are bitwise what they are without it."""
    from vmap_b200.track import SampleGroup, track_samples
    sg, og = _group(32, 3, 40, 10, seed=31)
    og["batch"]["sem"][1] = 2
    og["batch"]["mask_depth"][1] = False
    sg3 = SampleGroup(sg.ens, sg.active, og["batch"], 1)
    T = _rand_pose(8)
    out = track_samples([sg3], T, 1, 0.0, 0.0)
    lt = sg3.loss_terms.cpu()
    assert float(lt[1, 0]) == 0.0 and float(lt[1, 2]) == 0.0 and float(lt[1, 1]) > 0.0
    rest = {k: v[[0, 2]] for k, v in og["batch"].items()}
    sg2 = SampleGroup(sg.ens, [sg.active[0], sg.active[2]], rest, 1)
    track_samples([sg2], T, 1, 0.0, 0.0)
    assert torch.equal(sg2.loss_terms.cpu(), lt[[0, 2]])
    loss, g, abs_sum, terms = to.evaluate([og], T)
    _check_grad(out["grad_hist"][0].cpu().numpy(), g, abs_sum)
    _check_terms(lt.double().numpy(), terms[0].numpy())


def _scene(device="cuda:0"):
    """A 64 x 48 frame of three instances in front of a background, ingested into a FrameStore, and small random maps
    for the objects (hidden 32) and the background (hidden 128)."""
    from vmap_b200.cfg import Config, replica_room0_dict
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.keyframes import FrameStore
    d = replica_room0_dict()
    d["camera"].update(w=64, h=48, fx=40.0, fy=40.0, cx=31.5, cy=23.5)
    cfg = Config(config_dict=d)
    W, H = cfg.W, cfg.H
    g = torch.Generator().manual_seed(0)
    inst = torch.zeros(W, H, dtype=torch.int32)
    inst[5:25, 5:30] = 1
    inst[30:50, 10:40] = 2
    inst[40:60, 2:20] = 3
    inst[0:3, :] = -1
    depth = 1.0 + torch.rand(W, H, generator=g) * 2.0
    depth[::7, ::5] = 0.0
    rgb = torch.randint(0, 256, (W, H, 3), generator=g, dtype=torch.uint8)
    store = FrameStore(W, H, 4, device=device, max_id=16)
    slot, _, _ = store.ingest(rgb, depth, inst, torch.eye(4), min_extent=2)
    objs = VmapEnsemble(4, hidden=32, scale=2.0, impl="fp32")
    objs.load_stacked(vo.init_params(4, 32, seed=1))
    bg = VmapEnsemble(1, hidden=128, scale=5.0, impl="fp32")
    bg.load_stacked(vo.init_params(1, 128, seed=2))
    groups = [(objs, [1, 2, None, 3]), (bg, [0])]
    return cfg, store, slot, groups


def test_tracker_reproducible_and_graph_replay():
    from vmap_b200.track import Tracker
    cfg, store, slot, groups = _scene()
    T0 = _rand_pose(4, rot_deg=1.0, trans=0.02)
    kw = dict(n_iter=6, n_pix=40, n_pix_bg=120, seed=7)
    p1, l1 = Tracker(groups, cfg, **kw).track(store, slot, T0)
    assert torch.equal(store.t_wc[slot], p1.float())
    p2, l2 = Tracker(groups, cfg, **kw).track(store, slot, T0)
    assert torch.equal(p1, p2) and torch.equal(l1, l2)
    assert torch.all(torch.isfinite(l1)) and not torch.equal(p1.cpu(), torch.from_numpy(T0))
    t3 = Tracker(groups, cfg, **kw)
    t3.capture(store, slot, T0)
    p3, l3 = t3.run(store, slot, T0)
    assert torch.equal(p1, p3) and torch.equal(l1, l3)
    assert int(t3.status[0]) == 0


def _args(sg, n_iter=1, it=1):
    from vmap_b200 import _lib
    a = _lib.TrackArgs()
    a.n_groups, a.n_iter, a.iter = 1, n_iter, it
    pose = torch.eye(4, dtype=torch.float64, device="cuda:0")
    adam = torch.zeros(12, dtype=torch.float64, device="cuda:0")
    status = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    a.pose, a.adam, a.status = C.c_void_p(pose.data_ptr()), C.c_void_p(adam.data_ptr()), C.c_void_p(status.data_ptr())
    a.lr_rot = a.lr_trans = 1e-3
    a.beta1, a.beta2, a.eps = 0.9, 0.999, 1e-8
    a.colour_scaling, a.opacity_scaling = 5.0, 10.0
    sg.bind(a.group[0], 0)
    return a, (pose, adam, status)


def test_argument_checks():
    from vmap_b200 import _lib
    from vmap_b200.ensemble import _stream
    sg, _ = _group(32, 3, 20, 10, seed=41)
    L, h, st = sg.ens.lib, sg.ens._handle, _stream()

    def step(mut, group=0):
        a, keep = _args(sg)
        mut(a)
        return L.vmb_track_step(h, C.byref(a), group, st)

    def update(mut):
        a, keep = _args(sg)
        mut(a)
        return L.vmb_track_update(h, C.byref(a), st)

    assert step(lambda a: None) == 0
    assert update(lambda a: None) == 0
    E_ARG, E_UNS = -1, -4
    assert step(lambda a: setattr(a.group[0], "n_obj", 0)) == E_ARG
    assert step(lambda a: setattr(a.group[0], "n_rows", 0)) == E_ARG
    assert step(lambda a: setattr(a.group[0], "n_rays", 0)) == E_ARG
    assert step(lambda a: setattr(a.group[0], "rows", None)) == E_ARG
    assert step(lambda a: setattr(a.group[0], "hidden", 64)) == E_ARG
    assert step(lambda a: setattr(a.group[0], "max_partials", 1)) == E_ARG
    assert step(lambda a: setattr(a.group[0], "n_samples", 33)) == E_UNS
    assert step(lambda a: setattr(a, "n_iter", 0)) == E_ARG
    assert step(lambda a: setattr(a, "iter", 2)) == E_ARG
    assert step(lambda a: None, group=1) == E_ARG
    assert step(lambda a: setattr(a, "pose", None)) == E_ARG
    assert update(lambda a: setattr(a, "n_groups", 9)) == E_ARG
    assert update(lambda a: setattr(a, "lr_rot", -1.0)) == E_ARG
    assert update(lambda a: setattr(a, "lr_trans", float("nan"))) == E_ARG
    assert update(lambda a: setattr(a, "beta2", 1.0)) == E_ARG
    assert update(lambda a: setattr(a, "adam", None)) == E_ARG
    assert L.vmb_track_tiles(256, 10, 33) == E_UNS and L.vmb_track_tiles(48, 10, 10) == E_ARG
    torch.cuda.synchronize()


def test_device_side_guards():
    """A row outside the stack raises VMB_TRACK_ST_BAD_ROW; a non-finite pose skips the update and raises
    VMB_ST_NONFINITE, leaving the pose as it was."""
    from vmap_b200 import _lib
    from vmap_b200.ensemble import _stream
    sg, _ = _group(32, 2, 20, 10, seed=51)
    L, h, st = sg.ens.lib, sg.ens._handle, _stream()
    sg.rows_dev[1] = 99
    a, (pose, adam, status) = _args(sg)
    assert L.vmb_track_step(h, C.byref(a), 0, st) == 0
    assert L.vmb_track_update(h, C.byref(a), st) == 0
    assert int(status[0]) & _lib.TRACK_ST_BAD_ROW
    sg.rows_dev[1] = 2
    a, (pose, adam, status) = _args(sg)
    pose[0, 3] = float("nan")
    before = pose.clone()
    assert L.vmb_track_step(h, C.byref(a), 0, st) == 0
    assert L.vmb_track_update(h, C.byref(a), st) == 0
    assert int(status[0]) & _lib.VMB_ST_NONFINITE
    assert torch.equal(torch.isnan(pose), torch.isnan(before))
    assert torch.equal(torch.nan_to_num(pose), torch.nan_to_num(before))


def test_reference_golden():
    """The kernel against the reference's own UniDirsEmbed / OccupancyMap / step_batch_loss (tests/golden/ref_track.npz,
    oracle/make_track_golden.py): three hidden-32 objects and a hidden-128 background, each alone and both together."""
    import os
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.track import SampleGroup, track_samples
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_track.npz"))
    sgs, ogs = {}, {}
    for tag in ("obj", "bg"):
        params = {k: torch.from_numpy(g[f"{tag}_p_{k}"]) for k in vo.ALL_KEYS}
        batch = {k: torch.from_numpy(g[f"{tag}_in_{k}"]) for k in ("pcs", "z", "gt_depth", "gt_colour", "sem",
                                                                    "mask_depth")}
        B, hidden = batch["pcs"].shape[0], params["mid1.0.0.weight"].shape[1]
        ens = VmapEnsemble(B, hidden=hidden, scale=float(g[f"{tag}_scale"]), impl="fp32")
        ens.load_stacked({k: v.float() for k, v in params.items()})
        f32 = {k: (v.float() if v.is_floating_point() else v) for k, v in batch.items()}
        sgs[tag] = SampleGroup(ens, list(range(B)), f32, 1)
        ogs[tag] = {"params": {k: v.float() for k, v in params.items()},
                    "scale": torch.full((B,), float(g[f"{tag}_scale"])), "batch": f32}
        T = g[f"{tag}_pose"]
        out = track_samples([sgs[tag]], T, 1, 0.0, 0.0)
        loss_ref, grad_ref = float(g[f"{tag}_loss"]), g[f"{tag}_grad"]
        _, _, abs_sum, _ = to.evaluate([ogs[tag]], T)
        assert abs(float(out["losses"][0]) - loss_ref) <= 1e-5 * abs(loss_ref), tag
        _check_grad(out["grad_hist"][0].cpu().numpy(), grad_ref, abs_sum)


def test_graph_dropped_when_tracked_set_changes():
    """A graph writes into the buffers of the set it was captured for: tracking another set drops it, and run() then
    refuses instead of replaying into freed memory; capturing again works."""
    from vmap_b200 import _lib
    from vmap_b200.track import Tracker
    cfg, store, slot, groups = _scene()
    T0 = _rand_pose(4, rot_deg=1.0, trans=0.02)
    kw = dict(n_iter=4, n_pix=40, n_pix_bg=120, seed=3)
    tr = Tracker(groups, cfg, **kw)
    tr.capture(store, slot, T0, ids=[1, 2, 3])
    tr.track(store, slot, T0, ids=[1, 2])
    with pytest.raises(_lib.VmbError):
        tr.run(store, slot, T0)
    tr.capture(store, slot, T0, ids=[1, 2])
    p_graph, l_graph = tr.run(store, slot, T0)
    t2 = Tracker(groups, cfg, **kw)
    t2.track(store, slot, T0, ids=[1, 2])                   # the same draw counter as tr: one eager frame before
    p_eager, l_eager = t2.track(store, slot, T0, ids=[1, 2])
    assert torch.equal(p_graph, p_eager) and torch.equal(l_graph, l_eager)


def test_tracker_sampling_path():
    """Tracker's own samples: identity-pose camera points (z component equals the sample depth), object rays inside the
    object's ingest box and background rays over the full frame, the groups' bin counts, and the gradient of the first
    iteration equal to the oracle's on those very buffers."""
    from vmap_b200.track import Tracker
    cfg, store, slot, groups = _scene()
    T0 = _rand_pose(5, rot_deg=1.0, trans=0.02)
    tr = Tracker(groups, cfg, n_iter=3, n_pix=40, n_pix_bg=120, seed=1, record=True)
    tr.track(store, slot, T0)
    live = tr._live()
    assert [g.S for g in live] == [cfg.n_bins_cam2surface + cfg.n_bins, cfg.n_bins_cam2surface_bg + cfg.n_bins]
    ogs = []
    for g in live:
        o = {k: v[:, :g.n_pix].cpu() for k, v in g.out.items()}
        pcs = o["pcs"]
        assert torch.equal(pcs[..., 2], o["z"])
        zc = pcs[..., -1, 2]                                   # the deepest sample of each ray: z > 0
        assert bool((zc > 0).all())
        u = pcs[..., -1, 0] / zc * cfg.fx + cfg.cx
        v = pcs[..., -1, 1] / zc * cfg.fy + cfg.cy
        for k, r in enumerate(g.active):
            box = [0.0, cfg.W, 0.0, cfg.H] if g.bg else store.bbox[g.ids[r]].tolist()
            assert float(u[k].min()) >= box[0] - 1e-3 and float(u[k].max()) <= box[1] + 1e-3
            assert float(v[k].min()) >= box[2] - 1e-3 and float(v[k].max()) <= box[3] + 1e-3
        if not g.bg:
            assert bool((o["sem"] == 1).any(1).all())
        st = g.ens.stacked()
        ogs.append({"params": {k: t[g.active].cpu() for k, t in st.items()}, "scale": g.ens.scale[g.active].cpu(),
                    "batch": o})
    _, grad, abs_sum, _ = to.evaluate(ogs, tr.pose_hist[0].cpu().numpy())
    _check_grad(tr.grad_hist[0].cpu().numpy(), grad, abs_sum)


def test_skipped_first_iteration_restarts_the_moments():
    """Moments left by an earlier frame are cleared at iteration 1 even when that iteration's update is skipped."""
    from vmap_b200.ensemble import _stream
    sg, _ = _group(32, 2, 20, 10, seed=61)
    L, h, st = sg.ens.lib, sg.ens._handle, _stream()
    a, (pose, adam, status) = _args(sg)
    adam.fill_(0.5)
    pose[1, 3] = float("inf")
    assert L.vmb_track_step(h, C.byref(a), 0, st) == 0
    assert L.vmb_track_update(h, C.byref(a), st) == 0
    assert torch.equal(adam, torch.zeros_like(adam)) and int(status[0]) != 0
