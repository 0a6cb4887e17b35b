"""The joint map-and-pose step at hidden 32 (vmb_joint_step_fused: k_joint_world, k_step_fused<S, true>, k_joint_rows)
against the fp16-faithful restatement of oracle/joint_fused_oracle.py, which reads everything the kernel decides from
the kernel itself: its world points (pcs_world_out), its embedding of them (probe_embedding), its L1 signs and ray
variances (outputs=) and its mask counts.

The rows are compared per ray, per (object, frame) and through each object's loss terms, at every sample count the
launch instantiates (the S = 10 / 14 specialisations and the runtime-S kernel), with partial last tiles, CTAs that
run several tiles and per-object scales that are not powers of two; at later iterations, against the weights the
previous launch's fused AdamW left; at the bad-frame, empty-mask and all-terms-off edges; and against the exact fp64
model.  References that each carry one deliberate error show that the bars can see it.  test_joint_vmap_gpu.py
compares the same rows with K11 (fp32 network) and the fp64 oracle, at bars the fp16 network sets; here what is left is
fp32 accumulation order against fp64.

Run with -s to see every measured value next to its bar.
"""
import functools
import math

import numpy as np
import pytest
import torch

from oracle import fused_oracle as fo
from oracle import joint_fused_oracle as jfo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo
from oracle.lw_oracle import INV_LS
from tests.test_fused_faithful_gpu import loss_err, probe_embedding

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NPD = 10                                        # rays per draw
SEEDS = (0, 1, 2)
MAX_CTAS = 192                                  # k_step_fused.cuh's uf::MAX_CTAS

# Bars, 4-5x the worst an H100 80GB HBM3 (700 W power limit) measured over SHAPES and SEEDS (the tests print every
# value).  The row measures are taken over the rays without a forward flip (_forward_flips):
RAY_BAR = 1.7e-4        # per ray, max over the six components of sum |r - r_f| / sum |r_f|: worst 4.3e-5 (S 1, B 3)
OBJ_FRAME_BAR = 1.5e-3  # per (object, frame) gradient, max |g - g_f| / |g_f|: worst 3.1e-4 (S 2, B 1)
TERM_BAR = 1.5e-4       # per (object, loss term), test_fused_faithful_gpu.loss_err: worst 3.1e-5 (S 10, B 20)
# per frame over all objects against the exact fp64 model (ROUND_OFF on fp64 world points), max |g - g_x| / |g_x|:
# worst 6.1e-2 (S 5, B 3) with two or more samples per ray; 0.14 with one, where each ray's render is one fp16
# network output and nothing averages its error
EXACT_BAR, EXACT_BAR_S1 = 0.25, 0.6
# Forward flips: a ray whose render differs by more than FLIP_RENDER; measured at most 5 of 1,400 rays in one run
# (S 10, B 20) and 2 of 390 (S 1, B 3).  Allowed: the larger of 2 rays and FLIP_SHARE of the rays.
FLIP_RENDER = 1e-4
FLIP_SHARE = 0.01
# With the flips in, per ray reaches 1.9e-4 (S 32, B 20: one ray whose fc1 rounding flipped carries 91% of the sum).
# Each deliberate-error reference must fail RAY_BAR at one or more shapes.  Measured, kernel against it: dL/dt from the
# fp16 dproj 1.9e-4 .. 3.0e-4 (a factor 1.1 .. 1.8 over the bar: the fp16 rounding of dproj is the smallest error the
# per-ray measure resolves); direction 20 dropped 0.22 .. 0.42; object 0's scale 0.33 .. 0.76 at B > 1; rows moved by
# one ray 1.6 .. 1.9.


def _max_flips(n_rays):
    return max(2, int(FLIP_SHARE * n_rays))


# (S, B, R): every S instantiation, R never a multiple of the rays per tile 4 * (32 // S), B of 1, 3 and >= 20
SHAPES = [(1, 3, 130), (2, 1, 70), (5, 3, 50), (7, 20, 70), (10, 3, 70), (10, 20, 70), (14, 3, 70), (16, 1, 70),
          (17, 24, 90), (32, 20, 70)]
IDS = ["S{}B{}R{}".format(*c) for c in SHAPES]


def _rand_pose(seed, rot_deg=5.0, trans=0.05):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w * math.radians(rot_deg) / np.linalg.norm(w))
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _scales(B, seed):
    """Distinct per-object scales in [1.3, 3.7], none a power of two."""
    return torch.tensor(np.roll(np.linspace(1.3, 3.7, B), seed), dtype=torch.float32)


def _case(S, B, R, seed, n_iter=1):
    """A B-object hidden-32 stack at per-object scales, camera-frame samples of n_iter slices of R rays (every mask term
    on), draws of NPD rays alternating between two keyframe indices per object, and a 3-frame pose table."""
    from vmap_b200.ensemble import VmapEnsemble
    params = vo.init_params(B, 32, seed=seed)
    scale = _scales(B, seed)
    ens = VmapEnsemble(B, hidden=32, scale=scale, impl="umma")
    ens.load_stacked(params)
    batch = fo.synthetic(B, n_iter * R, S, seed + 1)
    n_draw = n_iter * R // NPD
    kf_draw = np.stack([(np.arange(n_draw) + b) % 2 for b in range(B)]).astype(np.int32)
    kf_frame = np.array([[[1, 2], [0, 2], [1, 0]][b % 3] for b in range(B)], np.int32)
    P = np.stack([np.eye(4), _rand_pose(seed + 2), _rand_pose(seed + 3)])
    return ens, params, scale, batch, kf_draw, kf_frame, P


def _frames(kf_draw, kf_frame, n_poses):
    """[B, rays] the pose-table row of each ray (-1 where the keyframe's frame is outside the table)."""
    f = np.stack([kf_frame[b][kf_draw[b]] for b in range(kf_draw.shape[0])])
    f = np.where((f >= 0) & (f < n_poses), f, -1)
    return torch.from_numpy(f.repeat(NPD, 1).astype(np.int64))


def _group(ens, batch, n_iter, kf_draw, kf_frame):
    from vmap_b200.ba import BaSampleGroup
    return BaSampleGroup(ens, list(range(ens.n_obj)), batch, n_iter, NPD, kf_draw, kf_frame)


def _args(g, P, n_iter, lr_rot=0.0, lr_trans=0.0, window=(1, 2)):
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


def _launch(ens, g, a, it):
    """Iteration ``it`` of the joint step (fused AdamW inside it): the rows [B,R,10], world points, render, loss terms
    and the slice's mask counts, on the host except the world points."""
    B, R, S = len(g.rows), g.n_pix, g.S
    f32 = dict(dtype=torch.float32, device=DEV)
    outs = {"depth": torch.empty(B, R, **f32), "var": torch.empty(B, R, **f32),
            "colour": torch.empty(B, R, 3, **f32), "opacity": torch.empty(B, R, **f32)}
    world = torch.empty(B, R, S, 3, **f32)
    a.iter = it + 1
    g.bind(a.group[0], it)
    g.ray_rows.fill_(float("nan"))
    sl = {k: v[:, it * R:(it + 1) * R] for k, v in g.out.items()}
    counts = ens.mask_counts(sl)
    ens.joint_step_fused(sl, a, 0, outputs=outs, pcs_world_out=world)
    torch.cuda.synchronize()
    return {"rows": g.ray_rows.view(B, R, 10).cpu().double(), "world": world,
            "render": {k: v.cpu() for k, v in outs.items()}, "terms": ens.loss_terms.cpu().double(),
            "counts": counts.cpu()}


def _slice(batch, it, R):
    return {k: v[:, it * R:(it + 1) * R].contiguous() for k, v in batch.items()}


def _reference(params, scale, sl, P, frames, kern, rounding=jfo.ROUND_ALL, kernel_inputs=True):
    """The restatement on the kernel's world points and embedding (``kernel_inputs``; otherwise its own world points
    and embedding), with the kernel's signs, variances and counts."""
    B, R, S, _ = sl["pcs"].shape
    o = kern["render"]
    signs = fo.signs_from_render(o["depth"], o["colour"], o["opacity"], sl)
    world = emb = None
    if kernel_inputs:
        world = kern["world"].cpu().double()
        e1, e2 = probe_embedding(params, scale, kern["world"].reshape(B, R * S, 3))
        emb = (e1.cpu(), e2.cpu())
    return jfo.evaluate(params, scale.double(), sl, P, frames, world=world, emb=emb, signs=signs, var=o["var"],
                        counts=kern["counts"], rounding=rounding)


def _forward_flips(kern, ref, z):
    """[B,R] rays whose kernel render already differs from the restatement's (from the same embedding) by more than
    FLIP_RENDER: depth relative to the ray's last z, opacity and colour absolutely.  There an fp16 rounding of the
    forward went the other way: a pre-activation within fp32 accumulation error of an fp16 midpoint (measured: fc1
    at 1.7e-8 of a midpoint, which moves the ray's opacity by the kernel's 8.9e-4).  Such a ray's row differs by as
    much as its forward does, so the row bars are taken over the other rays, and the flips are counted."""
    D, _, C, O = ref["render"]
    o = kern["render"]
    dev = torch.stack([(o["depth"].double() - D).abs() / z[..., -1].double(), (o["opacity"].double() - O).abs(),
                       (o["colour"].double() - C).abs().amax(-1)], -1).amax(-1)
    return dev > FLIP_RENDER, dev


def _ray_err(rows, ref, keep=None):
    """Per component c: sum over rays of |r_c - r_f,c| over sum of |r_f,c|; the largest of the six."""
    d, a = (rows[..., :6] - ref).abs(), ref.abs()
    d, a = (d[keep], a[keep]) if keep is not None else (d.reshape(-1, 6), a.reshape(-1, 6))
    return float((d.sum(0) / a.sum(0).clamp_min(1e-300)).max())


def _obj_frame_err(rows, ref, frames, keep=None):
    """Per (object, frame): max |g - g_f| / |g_f| of the rows summed over the rays of ``keep``.  A pair whose
    restated rows are all exactly zero (a fully opaque object with only its opacity term on) is left to the per-ray
    measure."""
    worst = 0.0
    for b in range(rows.shape[0]):
        for f in frames[b].unique().tolist():
            m = frames[b] == f
            if keep is not None:
                m &= keep[b]
            if f < 0 or not bool((ref[b, m] != 0).any()):
                continue
            gk, gr = rows[b, m, :6].sum(0), ref[b, m].sum(0)
            worst = max(worst, float((gk - gr).abs().max() / gr.norm()))
    return worst


def _frame_err(rows, grad, frames):
    gk = jfo.frame_grads(rows[..., :6], frames, grad.shape[0])
    return max(float((gk[f] - grad[f]).abs().max() / grad[f].norm()) for f in frames.unique().tolist() if f >= 0)


def _wrong_rows(ref, params, scale, sl, P, frames):
    """References that each carry one deliberate error."""
    q, dt, dproj = sl["pcs"], ref["dt"], ref["dproj"]
    dirs = params[vo.PE_KEY].double()
    B, R = frames.shape

    def rows(d, sc=scale):
        return jfo.pose_rows(d, sc.double(), q, P, frames)
    return {"dproj16": rows(dt + INV_LS * torch.matmul(fo._half(dproj, True) - dproj, dirs)),     # dL/dt from FG_DPR
            "dir20": rows(dt - INV_LS * dproj[..., 20:21] * dirs[:, None, 20]),                   # no hsel tail
            "scale0": rows(dt, scale[:1].expand(B)),                                              # object 0's scale
            "shift": ref["rows"].view(B, R // NPD, NPD, 6).roll(-1, 2).reshape(B, R, 6)}          # next ray's row


def _check_world(kern, P, frames, sl):
    """k_joint_world is pose_point at scale 1, bit for bit (a ray without a frame keeps its camera-frame point)."""
    want = jfo.world_points(P, frames, sl["pcs"])
    assert torch.equal(kern["world"].cpu().double(), want), "world points"


@functools.lru_cache(maxsize=None)
def _parity(S, B, R, seed):
    ens, params, scale, batch, kf_draw, kf_frame, P = _case(S, B, R, seed)
    g = _group(ens, batch, 1, kf_draw, kf_frame)
    a, k = _args(g, P, 1)
    kern = _launch(ens, g, a, 0)
    assert int(k["status"][0]) == 0
    assert bool(torch.isfinite(kern["rows"]).all()) and bool((kern["rows"][..., 6:] == 0).all())
    assert bool((kern["counts"][:, :3] > 0).all())                      # every loss term on
    frames = _frames(kf_draw, kf_frame, P.shape[0])
    _check_world(kern, P, frames, batch)
    ref = _reference(params, scale, batch, P, frames, kern)
    exact = _reference(params, scale, batch, P, frames, kern, rounding=jfo.ROUND_OFF, kernel_inputs=False)
    flip, dev = _forward_flips(kern, ref, batch["z"])
    keep = ~flip
    m = {"ray": _ray_err(kern["rows"], ref["rows"], keep), "ray_all": _ray_err(kern["rows"], ref["rows"]),
         "obj_frame": _obj_frame_err(kern["rows"], ref["rows"], frames, keep),
         "terms": loss_err(kern["terms"], ref["terms"]), "exact": _frame_err(kern["rows"], exact["grad"], frames),
         "flips": int(flip.sum()), "render": float(dev[keep].max())}
    assert m["flips"] <= _max_flips(B * R), m["flips"]
    for name, w in _wrong_rows(ref, params, scale, batch, P, frames).items():
        m["wrong_" + name] = _ray_err(kern["rows"], w, keep)
    return m


@pytest.mark.parametrize("S,B,R", SHAPES, ids=IDS)
def test_rows_against_the_restatement(S, B, R):
    worst = {}
    for seed in SEEDS:
        for key, v in _parity(S, B, R, seed).items():
            worst[key] = max(worst.get(key, 0.0), v)
    flips = sum(_parity(S, B, R, s)["flips"] for s in SEEDS)
    exact_bar = EXACT_BAR_S1 if S == 1 else EXACT_BAR
    print(f"\nS{S} B{B} R{R}: per ray {worst['ray']:.2e} (bar {RAY_BAR:.1e}), per (object, frame) "
          f"{worst['obj_frame']:.2e} (bar {OBJ_FRAME_BAR:.1e}), loss terms {worst['terms']:.2e} (bar {TERM_BAR:.1e}); "
          f"per frame vs exact fp64 {worst['exact']:.2e} (bar {exact_bar:.1e})")
    print(f"  forward flips {flips} of {len(SEEDS) * B * R} rays (at most {_max_flips(B * R)} per run); per ray with "
          f"them {worst['ray_all']:.2e}; largest render difference of the other rays {worst['render']:.2e} "
          f"(flip threshold {FLIP_RENDER:.0e})")
    print("  kernel vs the deliberate-error references, per ray (least over seeds): " + ", ".join(
        f"{n} {min(_parity(S, B, R, s)['wrong_' + n] for s in SEEDS):.2e}"
        for n in ("dproj16", "dir20", "scale0", "shift")))
    assert worst["ray"] <= RAY_BAR and worst["obj_frame"] <= OBJ_FRAME_BAR, worst
    assert worst["terms"] <= TERM_BAR and worst["exact"] <= exact_bar, worst


def test_the_bars_see_deliberate_errors():
    """Each deliberate error fails the per-ray bar at one or more committed shapes and seeds: dL/dt from the fp16
    dproj block instead of the fp32 dproj, the direction-20 (hsel tail) term dropped, object 0's scale in every
    object's rows, and each row moved to the next ray of its draw (the per-frame sums cannot see that one)."""
    for name in ("dproj16", "dir20", "scale0", "shift"):
        vals = {f"S{S}B{B}R{R}/{seed}": _parity(S, B, R, seed)["wrong_" + name] for S, B, R in SHAPES for seed in SEEDS}
        hi = max(vals, key=vals.get)
        lo = min(vals, key=vals.get)
        print(f"\n{name}: kernel vs that reference per ray, largest {vals[hi]:.2e} at {hi}, least {vals[lo]:.2e} at "
              f"{lo} (bar {RAY_BAR:.1e})")
        assert vals[hi] > RAY_BAR, name


def _cta_tiles(B, tpo, G):
    """Tiles per CTA of k_step_fused.cuh's fused_partition (the cost-aware split of B objects x tpo tiles over G)."""
    T = B * tpo
    rounds = -(-T // G)
    for beta in (1.0, 0.7, 0.4, 0.0):
        if beta > 0.0 and T < 2 * G:
            continue
        x = lambda t: t + beta * (t // tpo)            # noqa: E731
        begin = [0] * (G + 1)
        begin[G] = T
        most = 0
        for c in range(G - 1, 0, -1):
            end = begin[c + 1]
            top = x(end - 1) + 1.0
            cap = math.ceil(top / (c + 1) - 1e-9)
            p = end - 1
            while p - 1 >= c and top - x(p - 1) <= cap:
                p -= 1
            begin[c] = p
            most = max(most, end - p)
        most = max(most, begin[1])
        if most <= rounds:
            break
    return [begin[c + 1] - begin[c] for c in range(G)]


def test_shapes_cover_partial_tiles_and_multi_tile_ctas():
    """The launch's tiles B * ceil(R / nr) over a grid of min(tiles, SMs, MAX_CTAS): every shape ends each object on
    a partial tile, and one or more shapes give every CTA two or more tiles."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    fewest = []
    for S, B, R in SHAPES:
        nr = 4 * (32 // S)
        tpo = -(-R // nr)
        G = max(1, min(B * tpo, n_sm, MAX_CTAS))
        per = _cta_tiles(B, tpo, G)
        assert R % nr != 0 and sum(per) == B * tpo
        fewest.append(min(per))
        print(f"S{S} B{B} R{R}: {B * tpo} tiles of {nr} rays over {G} CTAs, {min(per)} .. {max(per)} per CTA")
    assert max(fewest) >= 2


@pytest.mark.parametrize("S", [7, 10])
def test_later_iterations_use_the_weights_adamw_left(S):
    """Three slices with the fused AdamW and nonzero pose rates: each launch's rows match the restatement at that
    launch's own weights, poses, samples and draw tables, and not at the previous launch's weights."""
    from vmap_b200.ba import ba_update
    B, R, n_iter = 3, 50, 3
    ens, params, scale, batch, kf_draw, kf_frame, P = _case(S, B, R, seed=5, n_iter=n_iter)
    ens.lr = 1e-2
    g = _group(ens, batch, n_iter, kf_draw, kf_frame)
    a, k = _args(g, P, n_iter, lr_rot=1e-3, lr_trans=1e-3)
    frames_all = _frames(kf_draw, kf_frame, P.shape[0])
    prev = None
    for it in range(n_iter):
        p_now = {kk: v.detach().cpu().clone() for kk, v in ens.stacked(ens.params).items()}
        P_now = k["poses"].cpu().numpy().copy()
        kern = _launch(ens, g, a, it)
        assert int(k["status"][0]) == 0
        ba_update(ens, a)
        sl, fr = _slice(batch, it, R), frames_all[:, it * R:(it + 1) * R]
        _check_world(kern, P_now, fr, sl)
        ref = _reference(p_now, scale, sl, P_now, fr, kern)
        flip, _ = _forward_flips(kern, ref, sl["z"])
        keep = ~flip
        e = _ray_err(kern["rows"], ref["rows"], keep)
        e_of, e_t = _obj_frame_err(kern["rows"], ref["rows"], fr, keep), loss_err(kern["terms"], ref["terms"])
        msg = (f"S{S} iteration {it + 1}: per ray {e:.2e} (bar {RAY_BAR:.1e}), per (object, frame) {e_of:.2e}, terms "
               f"{e_t:.2e}, forward flips {int(flip.sum())}")
        assert int(flip.sum()) <= _max_flips(flip.numel())
        if prev is not None:
            stale = _ray_err(kern["rows"], _reference(prev, scale, sl, P_now, fr, kern)["rows"], keep)
            msg += f"; against the previous launch's weights {stale:.2e}"
            assert stale > RAY_BAR, it
        print(msg)
        assert e <= RAY_BAR and e_of <= OBJ_FRAME_BAR and e_t <= TERM_BAR, (it, e, e_of, e_t)
        prev = p_now
    assert not np.array_equal(k["poses"].cpu().numpy(), P)


def test_bad_frame_rays():
    """Object 0's keyframe index 1 names no frame: its rays in those draws keep their camera-frame points and get
    exactly zero rows; the object's other rays, and the other objects, still match the restatement."""
    from vmap_b200 import _lib
    S, B, R = 7, 3, 70
    ens, params, scale, batch, kf_draw, kf_frame, P = _case(S, B, R, seed=9)
    kf_frame[0, 1] = 7
    g = _group(ens, batch, 1, kf_draw, kf_frame)
    a, k = _args(g, P, 1)
    kern = _launch(ens, g, a, 0)
    assert int(k["status"][0]) & _lib.BA_ST_BAD_FRAME
    frames = _frames(kf_draw, kf_frame, P.shape[0])
    bad = frames < 0
    assert bool(bad[0].any()) and not bool(bad[1:].any())
    assert bool((kern["rows"][bad] == 0).all())
    _check_world(kern, P, frames, batch)
    ref = _reference(params, scale, batch, P, frames, kern)
    flip, _ = _forward_flips(kern, ref, batch["z"])
    keep = ~bad & ~flip
    assert int(flip.sum()) <= _max_flips(flip.numel())
    e_all = _ray_err(kern["rows"], ref["rows"], keep=keep)
    e_0 = _ray_err(kern["rows"][:1], ref["rows"][:1], keep=keep[:1])
    print(f"\nbad-frame draws: per ray over the rays with a frame {e_all:.2e}, object 0's {e_0:.2e} "
          f"(bar {RAY_BAR:.1e})")
    assert e_all <= RAY_BAR and e_0 <= RAY_BAR


def test_empty_mask_object():
    """Object 1 has no object pixel: the mapping loss turns depth and colour off for every object, and each object's
    rows (opacity only) match the restatement, which applies that whole-batch rule."""
    S, B, R = 17, 3, 50
    ens, params, scale, batch, kf_draw, kf_frame, P = _case(S, B, R, seed=4)
    batch["sem"][:] = 1
    batch["sem"][1] = 0
    g = _group(ens, batch, 1, kf_draw, kf_frame)
    a, k = _args(g, P, 1)
    kern = _launch(ens, g, a, 0)
    assert int(k["status"][0]) == 0
    assert bool((kern["terms"][:, :2] == 0).all()) and bool((kern["terms"][:, 2] > 0).all())
    frames = _frames(kf_draw, kf_frame, P.shape[0])
    ref = _reference(params, scale, batch, P, frames, kern)
    flip, _ = _forward_flips(kern, ref, batch["z"])
    keep = ~flip
    assert int(flip.sum()) <= _max_flips(flip.numel())
    e, e_of = _ray_err(kern["rows"], ref["rows"], keep), _obj_frame_err(kern["rows"], ref["rows"], frames, keep)
    e_t = loss_err(kern["terms"], ref["terms"])
    print(f"\nempty-mask object: per ray {e:.2e} (bar {RAY_BAR:.1e}), per (object, frame) {e_of:.2e} "
          f"(bar {OBJ_FRAME_BAR:.1e}), terms {e_t:.2e} (bar {TERM_BAR:.1e})")
    assert e <= RAY_BAR and e_of <= OBJ_FRAME_BAR and e_t <= TERM_BAR


def test_every_term_off():
    """Only unknown pixels, and one object without object pixels: the whole-batch rule turns every term off, and the
    kernel's rows and the restatement's are exactly zero."""
    S, B, R = 5, 3, 50
    ens, params, scale, batch, kf_draw, kf_frame, P = _case(S, B, R, seed=6)
    batch["sem"][:] = 2
    batch["sem"][1] = 0
    g = _group(ens, batch, 1, kf_draw, kf_frame)
    a, k = _args(g, P, 1)
    kern = _launch(ens, g, a, 0)
    assert int(k["status"][0]) == 0
    frames = _frames(kf_draw, kf_frame, P.shape[0])
    ref = _reference(params, scale, batch, P, frames, kern)
    assert bool((kern["terms"] == 0).all()) and bool((ref["terms"] == 0).all())
    assert bool((kern["rows"] == 0).all()) and bool((ref["rows"] == 0).all())
