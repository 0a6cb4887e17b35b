"""The joint map-and-pose step at hidden 32 (vmb_joint_step_fused, FrameLoop's joint mode with a Background,
Slam(joint_poses=True, joint_impl="fused")): its per-ray pose rows against K11 and the fp64 oracle, the unchanged weight
path bit for bit, the update order, reproducibility, graph replay, the bad-frame rule, both groups of a background run
and vMAP SLAM end to end."""
import math

import numpy as np
import pytest
import torch

from oracle import ba_oracle as bo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NPD = 10                                        # rays per draw
R = 70                                          # not a multiple of the fused step's rays per tile (12 at S 10, 8 at S 14)


def _rand_pose(seed, rot_deg=5.0, trans=0.05):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    w *= math.radians(rot_deg) / np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w)
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _case(B, S, seed, n_iter=1, empty=None):
    """A B-object hidden-32 stack, camera-frame samples of n_iter slices of R rays and a 3-frame pose table; draws of NPD
    rays alternate between two keyframe indices naming frames (1, 2), (0, 2), (1, 0), ...  ``empty``: an object whose
    slice holds no object pixel (sem 0 everywhere)."""
    from vmap_b200.ba import BaSampleGroup
    from vmap_b200.ensemble import VmapEnsemble
    params = vo.init_params(B, 32, seed=seed)
    ens = VmapEnsemble(B, hidden=32, scale=2.0, impl="umma")
    ens.load_stacked(params)
    batch = vo.synthetic_batch(B, n_iter * R, S, seed=seed + 1, n_cam2surf=S - 9 if S > 9 else 1,
                               empty_prob=(0.0, 0.0, 0.0, 0.0))
    if empty is not None:
        batch["sem"][empty] = 0
    n_draw = n_iter * R // NPD
    kf_draw = np.stack([(np.arange(n_draw) + b) % 2 for b in range(B)]).astype(np.int32)
    kf_frame = np.array([[[1, 2], [0, 2], [1, 0]][b % 3] for b in range(B)], np.int32)
    P = np.stack([np.eye(4), _rand_pose(seed + 2), _rand_pose(seed + 3)])
    g = BaSampleGroup(ens, list(range(B)), batch, n_iter, NPD, kf_draw, kf_frame)
    frames = torch.from_numpy(np.stack([kf_frame[b][kf_draw[b]] for b in range(B)]).repeat(NPD, 1).astype(np.int64))
    og = {"params": params, "scale": torch.full((B,), 2.0), "batch": dict(batch, frames=frames)}
    return ens, g, P, og


def _fresh(og):
    from vmap_b200.ensemble import VmapEnsemble
    e = VmapEnsemble(og["scale"].numel(), hidden=32, scale=2.0, impl="umma")
    e.load_stacked(og["params"])
    return e


def _args(g, P, n_iter=1, lr_rot=0.0, lr_trans=0.0, window=(1, 2)):
    from vmap_b200.ba import ba_args
    f64 = dict(dtype=torch.float64, device=DEV)
    k = {"poses": torch.as_tensor(P, dtype=torch.float64).to(DEV).contiguous(),
         "win": torch.tensor(list(window), dtype=torch.int32, device=DEV),
         "adam": torch.zeros(len(window), 12, **f64),
         "scratch": torch.zeros(8 * len(g.rows) * g.win + 6 * len(window), **f64),
         "status": torch.zeros(4, dtype=torch.int32, device=DEV)}
    a = ba_args([g], n_iter, k["poses"], k["win"], len(window), 0, k["adam"], k["scratch"], lr_rot, lr_trans, None,
                k["status"])
    return a, k


def _slice(g, it):
    n = g.n_pix
    return {k: v[:, it * n:(it + 1) * n] for k, v in g.out.items()}


def _joint_rows(ens, g, P, fuse_adam=True):
    a, k = _args(g, P)
    a.iter = 1
    g.bind(a.group[0], 0)
    g.ray_rows.fill_(float("nan"))
    ens.joint_step_fused(_slice(g, 0), a, 0, fuse_adam=fuse_adam)
    torch.cuda.synchronize()
    return g.ray_rows.view(len(g.rows), -1, 10).cpu().numpy().copy(), k


def _ba_rows(g, P):
    """K11 (vmb_ba_step, hidden 32, fp32 CUDA cores) on the same samples and draw tables, at the ensemble's weights."""
    from vmap_b200.ba import ba_samples
    ba_samples([g], P, [1, 2], 1, 0.0, 0.0)
    torch.cuda.synchronize()
    return g.ray_rows.view(len(g.rows), -1, 10).cpu().numpy().copy()


def _rel(r, ref):
    """Summed per-component error over sum |ref| (the BA-row measure of test_joint_gpu.py)."""
    return float(np.abs(r[:, :, :6] - ref[:, :, :6]).sum((0, 1)).max() / np.abs(ref[:, :, :6]).sum())


def _per_frame_err(rows, og, P):
    _, grad, _, _ = bo.evaluate([og], P)
    fr = og["batch"]["frames"].numpy()
    return max(np.abs(rows[:, :, :6][fr == f].sum(0) - grad[f]).max() / np.linalg.norm(grad[f])
               for f in range(3) if (fr == f).any())


# Bars, about 4-5x the worst values an H100 (700 W) measured over the shapes below (the test prints them).  The fused
# step runs the network in fp16 on the tensor cores, K11 in fp32 on the CUDA cores: the rows differ by the fp16 rounding.
# Measured worst over S 10 / 14, B 1 / 3 / 20, two seeds each: 1.2e-3 against K11 and 0.12 per frame against the oracle
# (S 14, B 20); 3.5e-4 .. 9.3e-4 and 5e-3 .. 1.9e-2 at the other shapes.
JOINT32_BA_BAR = 5e-3            # against vmb_ba_step (K11, hidden 32), the _rel measure
JOINT32_ORACLE_BAR = 0.5         # per-frame sums against the fp64 ba_oracle, relative to the frame's gradient norm


@pytest.mark.parametrize("S,B", [(10, 1), (10, 3), (14, 3), (10, 20), (14, 20)])
def test_rows_against_k11_and_the_oracle(S, B):
    worst = [0.0, 0.0]
    for seed in (0, 1):
        ens, g, P, og = _case(B, S, seed=S + B + 10 * seed)
        r_b = _ba_rows(g, P)
        r_j, k = _joint_rows(ens, g, P)
        assert int(k["status"][0]) == 0
        assert np.all(np.isfinite(r_j)) and np.all(r_j[:, :, 6:] == 0.0)       # no loss columns
        worst = [max(worst[0], _rel(r_j, r_b)), max(worst[1], _per_frame_err(r_j, og, P))]
    print(f"S{S} B{B}: fused joint rows vs K11 {worst[0]:.2e}, per-frame vs fp64 oracle {worst[1]:.2e}")
    assert worst[0] <= JOINT32_BA_BAR and worst[1] <= JOINT32_ORACLE_BAR, worst


def test_rows_of_an_empty_mask_object():
    """The rows are the mapping loss's gradient, so its whole-batch rule holds: a term is off for every object when one
    object's count of it is 0 (K11 applies the rule per object).  Every other object's rays are object pixels here, so
    the empty object (sem 0: no depth or colour pixel) turns depth and colour off for all, and opacity stays on for
    all: the empty object's own loss is the same under both rules, and its rows are K11's and the fp64 oracle's."""
    ens, g, P, og = _case(3, 10, seed=4)
    g.out["sem"].fill_(1)
    g.out["sem"][1] = 0
    og["batch"]["sem"][:] = 1
    og["batch"]["sem"][1] = 0
    r_b = _ba_rows(g, P)
    r_j, k = _joint_rows(ens, g, P)
    assert int(k["status"][0]) == 0 and np.all(np.isfinite(r_j)) and np.abs(r_j[:, :, :6]).sum() > 0
    o1 = {"params": {kk: v[1:2] for kk, v in og["params"].items()}, "scale": og["scale"][1:2],
          "batch": {kk: v[1:2] for kk, v in og["batch"].items()}}
    e_b, e_o = _rel(r_j[1:2], r_b[1:2]), _per_frame_err(r_j[1:2], o1, P)
    print(f"empty-mask object: fused joint rows vs K11 {e_b:.2e}, per frame vs the fp64 oracle {e_o:.2e}")
    assert e_b <= JOINT32_BA_BAR and e_o <= JOINT32_ORACLE_BAR


def test_rows_are_zero_when_every_term_is_off():
    """_case's objects hold only unknown pixels (sem 2: no opacity pixel); with one object emptied of object pixels too,
    the whole-batch rule turns all three terms off: zero loss and exactly zero rows, where K11 keeps the empty
    object's opacity term and the others' depth and colour terms."""
    ens, g, P, og = _case(3, 10, seed=4, empty=1)
    r_j, k = _joint_rows(ens, g, P)
    assert int(k["status"][0]) == 0
    assert torch.equal(ens.loss_terms.cpu(), torch.zeros_like(ens.loss_terms.cpu()))
    assert np.all(r_j == 0.0)


def test_weight_path_bitwise_at_pose_rates_zero():
    """N joint iterations at pose rates 0 give the plain fused step's bits on the world points they return: the
    step kernel is the same code with a side output, and neither has floating-point atomics."""
    from vmap_b200.ba import ba_update
    n_iter, B, S = 6, 3, 10
    ens, g, P, og = _case(B, S, seed=7, n_iter=n_iter)
    world = [torch.empty(B, R, S, 3, dtype=torch.float32, device=DEV) for _ in range(n_iter)]
    a, k = _args(g, P, n_iter)
    f32 = dict(dtype=torch.float32, device=DEV)

    def outs():
        return {"depth": torch.empty(B, R, **f32), "var": torch.empty(B, R, **f32),
                "colour": torch.empty(B, R, 3, **f32), "opacity": torch.empty(B, R, **f32)}
    out_j, loss_j = outs(), torch.zeros(n_iter, **f32)
    terms_j = []
    for it in range(n_iter):
        a.iter = it + 1
        g.bind(a.group[0], it)
        ens.joint_step_fused(_slice(g, it), a, 0, outputs=out_j if it == 0 else None, loss_out=loss_j[it:it + 1],
                             pcs_world_out=world[it])
        terms_j.append(ens.loss_terms.clone())
        ba_update(ens, a)
    torch.cuda.synchronize()
    assert torch.equal(k["poses"].cpu(), torch.as_tensor(P))
    e = _fresh(og)
    out_p, loss_p = outs(), torch.zeros(n_iter, **f32)
    for it in range(n_iter):
        b = {kk: v[:, it * R:(it + 1) * R] for kk, v in g.out.items()}
        b["pcs"] = world[it]
        e.forward_backward(b, outputs=out_p if it == 0 else None, fuse_adam=True, loss_out=loss_p[it:it + 1])
        assert torch.equal(e.loss_terms, terms_j[it]), it
    torch.cuda.synchronize()
    for name in ("params", "exp_avg", "exp_avg_sq", "image", "step_counter"):
        assert torch.equal(getattr(ens, name), getattr(e, name)), name
    for kk in out_j:
        assert torch.equal(out_j[kk], out_p[kk]), kk
    assert torch.equal(loss_j, loss_p)


def test_rows_fuse_adam_update_order_reproducibility_and_graph():
    B, S = 3, 14
    ens, g, P, og = _case(B, S, seed=11)
    r_b = _ba_rows(g, P)
    r0, _ = _joint_rows(_fresh(og), g, P, fuse_adam=False)
    r0b, _ = _joint_rows(_fresh(og), g, P, fuse_adam=False)
    assert np.array_equal(r0, r0b)                                        # bitwise reproducible
    ens.lr = 1e-2                                                        # a step large enough to move K11's rows
    r1, _ = _joint_rows(ens, g, P, fuse_adam=True)
    assert np.array_equal(r0, r1)                                        # AdamW inside the step: the same rows
    r_after = _ba_rows(g, P)
    e_ok, e_late = _rel(r1, r_b), _rel(r1, r_after)
    print(f"fused joint rows vs K11 before the update {e_ok:.2e}, after it {e_late:.2e}")
    assert e_ok < e_late
    # graph replay = eager
    e2 = _fresh(og)
    a, k = _args(g, P)
    a.iter = 1
    g.bind(a.group[0], 0)
    e2.joint_step_fused(_slice(g, 0), a, 0, fuse_adam=False)           # warm-up (kernel attributes, workspace)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        e2.joint_step_fused(_slice(g, 0), a, 0, fuse_adam=False)
    g.ray_rows.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(g.ray_rows.view(B, -1, 10).cpu().numpy(), r0)


def test_bad_frame_and_guards():
    from vmap_b200 import _lib
    ens, g, P, og = _case(2, 10, seed=3)
    good, _ = _joint_rows(_fresh(og), g, P, fuse_adam=False)
    g.kf_frame[0, 1] = 7                                                 # object 0's keyframe index 1: no such frame
    bad_rows, k = _joint_rows(ens, g, P, fuse_adam=False)
    assert int(k["status"][0]) & _lib.BA_ST_BAD_FRAME
    bad = np.zeros(R, bool)
    for d in range(R // NPD):
        if d % 2 == 1:
            bad[d * NPD:(d + 1) * NPD] = True
    assert np.all(bad_rows[0, bad] == 0.0) and np.abs(bad_rows[0, ~bad, :6]).sum() > 0
    assert np.abs(bad_rows[1, :, :6]).sum() > 0
    # a group that does not describe the step's rays; a hidden-64 ensemble (it takes vmb_joint_step_lw)
    a, _ = _args(g, P)
    a.iter = 1
    g.bind(a.group[0], 0)
    a.group[0].n_rays = 30
    with pytest.raises(_lib.VmbError, match=r"\(-1\)"):
        ens.joint_step_fused(_slice(g, 0), a, 0)
    from vmap_b200.ba import BaSampleGroup
    from vmap_b200.ensemble import VmapEnsemble
    e64 = VmapEnsemble(1, hidden=64, scale=2.0, impl="layerwise")
    e64.load_stacked(vo.init_params(1, 64, seed=1))
    batch = vo.synthetic_batch(1, 20, 10, seed=2)
    g64 = BaSampleGroup(e64, [0], batch, 1, NPD, np.zeros((1, 2), np.int32), np.array([[1]], np.int32))
    a, _ = _args(g64, np.stack([np.eye(4)] * 2), window=(1,))
    a.iter = 1
    g64.bind(a.group[0], 0)
    with pytest.raises(_lib.VmbError):
        e64.joint_step_fused(_slice(g64, 0), a, 0)


# ---- vMAP: joint poses in Slam on the synthetic sphere room at 160 x 120 (test_slam_gpu.py's configuration) ----------
W, H, FX = 160, 120, 120.0
N = 24
SLAM_ATE_BAR = 0.03                              # test_slam_gpu.py's bar


def _cfg(do_bg=False):
    from vmap_b200.cfg import Config, replica_room0_dict
    d = replica_room0_dict()
    d["camera"].update(w=W, h=H, fx=FX, fy=FX, cx=W / 2 - 0.5, cy=H / 2 - 0.5)
    d["trainer"]["do_bg"] = int(do_bg)
    return Config(config_dict=d)


@pytest.fixture(scope="module")
def seq():
    from vmap_b200 import synth
    return synth.sphere_room_sequence(N, W, H, FX, FX, W / 2 - 0.5, H / 2 - 0.5)


def _run(seq, n=N, poses=None, do_bg=False, **kw):
    import random
    from vmap_b200.slam import Slam
    torch.manual_seed(0)
    random.seed(0)
    slam = Slam(_cfg(do_bg), T_init=seq["poses"][0], background_cls=seq["background_cls"], **kw)
    for k in range(n):
        slam.step(torch.from_numpy(seq["rgb"][k]), torch.from_numpy(seq["depth"][k].astype(np.float32)),
                  torch.from_numpy(seq["inst"][k]), torch.from_numpy(seq["cls"][k]),
                  T_wc=(poses if poses is not None else seq["poses"])[k])
    torch.cuda.synchronize()
    return slam


def _err(T, G):
    return float(np.linalg.norm(T[:3, 3] - G[:3, 3])), to.rot_err_deg(T[:3, :3], G[:3, :3])


def _noisy(seq):
    rng = np.random.default_rng(12)
    P = seq["poses"].copy()
    for k in range(1, N):
        w = rng.normal(size=3)
        t = rng.normal(size=3)
        P[k, :3, :3] = to.exp_so3_np(w * math.radians(3.0) / np.linalg.norm(w)) @ P[k, :3, :3]
        P[k, :3, 3] += 0.05 * t / np.linalg.norm(t)
    return P


@pytest.mark.parametrize("do_bg", [False, True])
def test_joint_poses_reduce_keyframe_noise(seq, do_bg):
    noisy = _noisy(seq)
    slam = _run(seq, poses=noisy, do_bg=do_bg, track=False, joint_poses=True, joint_impl="fused", seed=2)
    res = slam.result()
    assert np.array_equal(res["poses"][0], seq["poses"][0])
    before = np.array([_err(noisy[k], seq["poses"][k]) for k in range(1, N)])
    after = np.array([_err(res["poses"][k], seq["poses"][k]) for k in range(1, N)])
    print(f"vMAP joint poses (do_bg {do_bg}) from 5 cm / 3 deg keyframe noise: translation mean "
          f"{before[:, 0].mean() * 100:.2f} -> {after[:, 0].mean() * 100:.2f} cm, rotation mean "
          f"{before[:, 1].mean():.2f} -> {after[:, 1].mean():.2f} deg")
    assert after[:, 0].mean() < before[:, 0].mean() and after[:, 1].mean() < before[:, 1].mean()
    # the refined poses reached the store's slots and, with a background, its keyframe copies
    poses = torch.as_tensor(res["poses"], dtype=torch.float64)
    for o in slam.objects.values():
        for j in range(len(o._held)):
            if o._held[j]:
                s = o.kf_store_slot[j]
                f = int(slam.store.frame_id[s])
                assert torch.equal(slam.store.t_wc[s].cpu(), poses[f].float()), (o, j)
    if do_bg:
        loop = slam.loop
        assert loop.bg is not None
        for f, j in slam.scene_bg.kf_id_dict.items():
            if int(f) < res["poses"].shape[0] and int(f) in loop.pose_tables.window:
                assert torch.equal(slam.scene_bg.t_wc_batch[j].cpu(), poses[int(f)].float()), f
        for gr in (loop.jg, loop.jbg):                      # both groups' rows reached the update
            assert torch.isfinite(gr.ray_rows).all() and gr.ray_rows[:, :6].abs().sum() > 0


def test_vmap_slam_with_joint_poses(seq):
    from vmap_b200 import metrics
    ates, plain = [], []
    for seed in (2, 3, 4):
        res = _run(seq, track=True, graph=True, seed=seed, joint_poses=True, joint_impl="fused").result()
        assert not res["lost"].any() and np.isfinite(res["map_loss"]).all()
        ates.append(metrics.ate(res["poses"], seq["poses"])["rmse"])
        plain.append(metrics.ate(_run(seq, track=True, graph=True, seed=seed).result()["poses"], seq["poses"])["rmse"])
    print("vMAP SLAM ATE rmse (cm), seeds 2/3/4, joint poses: " + ", ".join(f"{a * 100:.3f}" for a in ates) +
          "; without: " + ", ".join(f"{a * 100:.3f}" for a in plain))
    assert max(ates) < SLAM_ATE_BAR


def test_joint_composes_with_ba_and_store_growth(seq):
    from vmap_b200 import metrics
    slam = _run(seq, n=12, track=True, graph=True, seed=2, joint_poses=True, joint_impl="fused", ba_every=4,
                store_capacity=2)
    res = slam.result()
    assert res["store_capacity"] > 2 and not res["lost"].any()
    assert slam.loop.graph is not None and slam.loop.pose_tables.cap == res["store_capacity"]
    assert any(m in ("eager", "capture", "replay") for m in res["ba_modes"])
    ate = metrics.ate(res["poses"], seq["poses"][:12])["rmse"]
    print(f"vMAP joint poses with BA every 4 and store growth from 2 slots: ATE rmse {ate * 100:.3f} cm over 12 frames")
    assert ate < SLAM_ATE_BAR
