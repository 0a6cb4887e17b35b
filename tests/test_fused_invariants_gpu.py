"""Checks of the hidden-32 fused step that the fp32-oracle bars cannot make, and of the per-object AdamW state and loss
guard on every path.

The oracle bars of test_umma_gpu.py / test_baseline_configs_gpu.py must absorb fp16-operand noise and L1 sign flips,
so a lost or double-counted tile, or a CTA's gradient partial reduced into the wrong row, stays inside them
(test_dropped_tile_is_rejected shows it). Here the kernel is compared with itself where the exact answer is known:
splitting the rays of a batch, permuting them, running an object alone, accumulating twice, and training the same
ensemble twice. The only difference left is the fp32 reassociation of the per-CTA gradient partials, so the bars are
per object and per tensor. AdamW is compared per object with torch.optim.AdamW in fp64, at step numbers on both sides
of the bias-correction table's edge. Run with -s to see every measured value next to its bar."""
import pytest
import torch

from oracle import vmap_oracle as vo
from tests._util import make_ensemble, rel_l2, to_dev

pytestmark = pytest.mark.gpu

# Bars: about four to five times the worst value measured (over SEEDS) on an H100 80GB HBM3 at a 700 W power limit.
BAR_INV_GRAD = 2e-5     # per (object, tensor) gradient rel-L2 between two arrangements of the same rays (worst 4.4e-6)
BAR_INV_LOSS = 1.5e-6   # per (object, term) relative loss-term difference (worst 3.4e-7)
# AdamW against torch.optim.AdamW in fp64, per object: the parameter UPDATE (p_new - p_old; worst 1.1e-5) and the
# moments (worst 2.5e-7)
BAR_ADAM_DELTA = 5e-5
BAR_ADAM_MOM = 1.2e-6
# loss guard: the surviving objects against a stack without the exploding one (reassociated gradient only; worst 5.8e-7)
BAR_GUARD = 2.5e-6

# the shapes of test_umma_gpu.test_oracle_parity_umma
SHAPES = [
    dict(B=4, R=301, S=10, n1=1),       # ragged last tile; CTAs straddle objects
    dict(B=5, R=30, S=10, n1=1),        # 3 tiles / object: every CTA spans two objects
    dict(B=2, R=100, S=14, n1=5),       # SC = 14 instantiation
    dict(B=1, R=64, S=16, n1=5),        # exactly 8 rays / tile, SC = 0 instantiation
    dict(B=3, R=40, S=1, n1=0),         # single sample per ray
    dict(B=2, R=33, S=20, n1=5),        # one ray per warp, 12 idle lanes
    dict(B=2, R=50, S=32, n1=8),        # 32 samples per ray
    dict(B=20, R=1200, S=10, n1=1),     # BASELINE cfg 2 at full size
]
IDS = ["B{B}R{R}S{S}".format(**c) for c in SHAPES]


def rays_per_tile(S):
    return 4 * (32 // S)


def make_batch(cfg, seed=11):
    B, R, S = cfg["B"], cfg["R"], cfg["S"]
    if S > 1:
        return vo.synthetic_batch(B, R, S, seed=seed, n_cam2surf=cfg["n1"])
    b2 = vo.synthetic_batch(B, R, 2, seed=seed, n_cam2surf=1)
    b2["pcs"], b2["z"] = b2["pcs"][:, :, :1].contiguous(), b2["z"][:, :, :1].contiguous()
    return b2


def rays(batch, sl):
    """Rays ``sl`` of every object (a strided view: each object's block stays dense)."""
    return {k: v[:, sl] for k, v in batch.items()}


def grads_of(ens, batch, counts=None):
    ens.grads.zero_()
    ens.forward_backward(batch, counts=counts)
    return ens.grads.clone(), ens.loss_terms.clone()


def grad_err(ens, got, ref):
    """Largest relative L2 error over (object, tensor) pairs of two packed gradient blocks, and where it is."""
    worst, where = 0.0, None
    for k in vo.ALL_KEYS:
        g = ens.view(k, got).double().flatten(1)
        r = ens.view(k, ref).double().flatten(1)
        num, den = (g - r).norm(dim=1), r.norm(dim=1)
        e = torch.where(den > 0, num / den.clamp_min(1e-300), num)        # an exactly-zero row must stay zero
        i = int(e.argmax())
        if float(e[i]) > worst or where is None:
            worst, where = float(e[i]), (i, k)
    return worst, where


def loss_err(got, ref):
    got, ref = got.double(), ref.double()
    return float(((got - ref).abs() / ref.abs().clamp_min(1e-30)).max())


def report(name, value, bar):
    print(f"  {name}: {value:.3e} (bar {bar:.1e})")
    return value


# ---- invariances of the fused kernel ------------------------------------------------------------------------------------

SEEDS = [11, 12, 13]


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("where", ["on_tile", "off_tile"])
@pytest.mark.parametrize("cfg", SHAPES, ids=IDS)
def test_ray_split_is_additive(cfg, where, seed):
    """forward_backward(A) + forward_backward(B) == forward_backward(A u B) with the full batch's mask counts; the
    loss terms add up and each ray renders to the same bits whichever sub-batch (and tile) it lands in."""
    R, nr = cfg["R"], rays_per_tile(cfg["S"])
    k = nr * max(1, (R // nr) // 2)
    if where == "off_tile":
        k = min(k + nr // 2 + 1, R - 1) if R > nr else R // 2
    if not 0 < k < R or (where == "on_tile" and k % nr):
        pytest.skip("no tile boundary inside the batch")
    params = vo.init_params(cfg["B"], 32, seed=seed - 4)
    db = to_dev(make_batch(cfg, seed))
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    counts = ens.mask_counts(db)
    g_full, l_full = grads_of(ens, db)
    ens.grads.zero_()
    ens.forward_backward(rays(db, slice(0, k)), counts=counts)
    l_a = ens.loss_terms.clone()
    ens.forward_backward(rays(db, slice(k, R)), counts=counts)
    l_b = ens.loss_terms.clone()
    ge, at = grad_err(ens, ens.grads, g_full)
    print(f"\nsplit at ray {k} of {R} ({where}), worst at {at}")
    assert report("grad", ge, BAR_INV_GRAD) < BAR_INV_GRAD, at
    assert report("loss terms", loss_err(l_a + l_b, l_full), BAR_INV_LOSS) < BAR_INV_LOSS
    full = ens.render(db)
    parts = [ens.render(rays(db, s)) for s in (slice(0, k), slice(k, R))]
    for f, a, b in zip(full, *parts):
        assert torch.equal(torch.cat([a, b], dim=1), f)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("cfg", SHAPES, ids=IDS)
def test_ray_permutation_within_objects(cfg, seed):
    """Shuffling each object's rays permutes the render outputs bit for bit and changes the gradient only by fp32
    reassociation of the per-CTA partials."""
    B, R = cfg["B"], cfg["R"]
    params = vo.init_params(B, 32, seed=seed - 4)
    db = to_dev(make_batch(cfg, seed))
    gen = torch.Generator().manual_seed(seed)
    idx = torch.stack([torch.randperm(R, generator=gen) for _ in range(B)]).cuda()
    dp = {k: torch.stack([v[b, idx[b]] for b in range(B)]).contiguous() for k, v in db.items()}
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    g0, l0 = grads_of(ens, db)
    g1, l1 = grads_of(ens, dp)
    ge, at = grad_err(ens, g1, g0)
    print(f"\npermuted rays, worst at {at}")
    assert report("grad", ge, BAR_INV_GRAD) < BAR_INV_GRAD, at
    assert report("loss terms", loss_err(l1, l0), BAR_INV_LOSS) < BAR_INV_LOSS
    for f, p in zip(ens.render(db), ens.render(dp)):
        assert torch.equal(torch.stack([f[b, idx[b]] for b in range(B)]), p)


@pytest.mark.parametrize("cfg", [c for c in SHAPES if c["B"] > 1], ids=[i for i, c in zip(IDS, SHAPES) if c["B"] > 1])
def test_object_isolation(cfg):
    """Each object of a stack gives what the same object gives alone (n_obj = 1): no CTA that straddles two objects
    leaks one object's rays or partial row into the other."""
    B = cfg["B"]
    params = vo.init_params(B, 32, seed=7)
    db = to_dev(make_batch(cfg))
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    g_all, l_all = grads_of(ens, db)
    r_all = ens.render(db)
    worst_g, worst_l = (0.0, None), 0.0
    for b in range(B):
        one = make_ensemble({k: v[b:b + 1] for k, v in params.items()}, 2.0, 32, impl="umma")
        db1 = {k: v[b:b + 1].contiguous() for k, v in db.items()}
        g1, l1 = grads_of(one, db1)
        e = grad_err(one, g_all[b:b + 1], g1)
        worst_g = max(worst_g, (e[0], (b, e[1][1])), key=lambda t: t[0])
        worst_l = max(worst_l, loss_err(l_all[b:b + 1], l1))
        for f, s in zip(r_all, one.render(db1)):
            assert torch.equal(f[b:b + 1], s)
    print(f"\nobjects alone vs in the stack, worst at {worst_g[1]}")
    assert report("grad", worst_g[0], BAR_INV_GRAD) < BAR_INV_GRAD, worst_g
    assert report("loss terms", worst_l, BAR_INV_LOSS) < BAR_INV_LOSS


@pytest.mark.parametrize("cfg", [SHAPES[0], SHAPES[7]], ids=[IDS[0], IDS[7]])
def test_gradient_accumulates_exactly(cfg):
    """Two forward_backward calls without a zero in between give exactly twice one call (the finisher adds the
    reduced gradient to ``grads`` once per object, padding columns stay zero)."""
    params = vo.init_params(cfg["B"], 32, seed=7)
    db = to_dev(make_batch(cfg))
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    g1, _ = grads_of(ens, db)
    ens.forward_backward(db)
    assert torch.equal(ens.grads, 2 * g1)
    assert float(g1[:, ens.count:].abs().sum()) == 0.0


def test_dropped_tile_is_rejected():
    """Power of the checks above, at BASELINE cfg 2: the full gradient minus one tile's rays of one object (a sub-batch
    run with the full counts -- exactly what a lost tile would give) fails the invariance bars by a wide margin, while
    the older fp32-oracle bars (test_umma_gpu: stack rel-L2 < 4e-2 and cosine > 0.999; test_baseline_configs_gpu:
    per-object max < 0.6) accept it."""
    cfg = SHAPES[7]
    B = cfg["B"]
    nr = rays_per_tile(cfg["S"])
    params = vo.init_params(B, 32, seed=7)
    batch = make_batch(cfg)
    db = to_dev(batch)
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    counts = ens.mask_counts(db)
    g_full, l_full = grads_of(ens, db)
    g_tile, l_tile = grads_of(ens, rays(db, slice(3 * nr, 4 * nr)), counts=counts)
    victim = 1
    g_bad = g_full.clone()
    g_bad[victim] -= g_tile[victim]
    l_bad = l_full.clone()
    l_bad[victim] -= l_tile[victim]
    ge, at = grad_err(ens, g_bad, g_full)
    print(f"\ntile 3 of object {victim} dropped, invariance comparator worst at {at}")
    report("grad (must FAIL the bar by 10x)", ge, BAR_INV_GRAD)
    report("loss terms (must FAIL the bar)", loss_err(l_bad, l_full), BAR_INV_LOSS)
    assert ge > 10 * BAR_INV_GRAD
    assert loss_err(l_bad, l_full) > BAR_INV_LOSS
    # the old bars, against the fp32 oracle
    orc = vo.OracleEnsemble(params, 2.0)
    _, g_ref = orc.grads(batch)
    worst_stack, worst_cos, worst_obj = 0.0, 1.0, 0.0
    for k in vo.ALL_KEYS:
        gb, gr = ens.view(k, g_bad).cpu(), g_ref[k]
        worst_stack = max(worst_stack, rel_l2(gb, gr))
        a, b = gb.double().flatten(), gr.double().flatten()
        worst_cos = min(worst_cos, float(a @ b / (a.norm() * b.norm())))
        per_obj = (gb - gr).double().flatten(1).norm(dim=1) / (gr.double().flatten(1).norm(dim=1) + 1e-20)
        worst_obj = max(worst_obj, float(per_obj.max()))
    print(f"  old bars: stack rel-L2 {worst_stack:.3e} (bar 4e-2), cosine {worst_cos:.6f} (bar 0.999), "
          f"per-object max {worst_obj:.3e} (bar 0.6)")
    assert worst_stack < 4e-2 and worst_cos > 0.999 and worst_obj < 0.6


# ---- reproducible finish -------------------------------------------------------------------------------------------------

def make_explode(params, batch, b):
    """Object b's depth loss exceeds 1e5: occupancy 1 at the first sample -> zero variance -> info weight 1e4."""
    params["out_alpha.bias"][b] += 50.0
    explode_batch(batch, b)


def explode_batch(batch, b):
    batch["z"][b] = 1.0
    batch["gt_depth"][b] = 1000.0
    batch["mask_depth"][b] = True
    batch["sem"][b] = 1


@pytest.mark.parametrize("explode", [False, True], ids=["clean", "object2_explodes"])
def test_finish_is_bitwise_reproducible(explode):
    """The grid-wide finish reduces the partial rows in segment order, whichever CTA reaches the grid barrier first,
    so two fresh ensembles trained for 50 steps on the same batches end with identical bits."""
    from vmap_b200.ensemble import LossExplode
    B, R, S = 7, 301, 10
    params = vo.init_params(B, 32, seed=3)
    batches = [vo.synthetic_batch(B, R, S, seed=50 + i) for i in range(4)]
    if explode:
        make_explode(params, batches[0], 2)
        for bt in batches[1:]:
            explode_batch(bt, 2)
    batches = [to_dev(bt) for bt in batches]
    runs = []
    for _ in range(2):
        ens = make_ensemble(params, 2.0, 32, impl="umma")
        losses = torch.stack([ens.step(batches[it % 4]) for it in range(50)])
        torch.cuda.synchronize()
        runs.append(dict(params=ens.params.clone(), exp_avg=ens.exp_avg.clone(), exp_avg_sq=ens.exp_avg_sq.clone(),
                         image=ens.image.clone(), step_counter=ens.step_counter.clone(),
                         loss_terms=ens.loss_terms.clone(), losses=losses))
        if explode:
            with pytest.raises(LossExplode):
                ens.check_status()
        else:
            ens.check_status()
    for k, v in runs[0].items():
        assert torch.equal(v, runs[1][k]), k
    want = torch.full((B,), 50, dtype=torch.int32, device="cuda")
    if explode:
        want[2] = 0
    assert torch.equal(runs[0]["step_counter"], want)


# ---- per-object AdamW state ----------------------------------------------------------------------------------------------

COUNTERS = [0, 1, 9, 20478, 20479, 20480, 40000]       # both sides of the 20480-entry bias-correction table


def set_random_state(ens, seed):
    gen = torch.Generator().manual_seed(seed)
    B, P = ens.n_obj, ens.count
    ens.exp_avg[:, :P] = (torch.randn(B, P, generator=gen) * 1e-2).cuda()
    ens.exp_avg_sq[:, :P] = (torch.rand(B, P, generator=gen) * 1e-4).cuda()
    ens.step_counter.copy_(torch.tensor(COUNTERS[:B], dtype=torch.int32))


def f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def torch_adamw(ens, p0, g, m0, v0, steps):
    """One torch.optim.AdamW step per object in fp64, object b resuming from step number steps[b]. The C ABI carries
    lr, betas, eps and weight decay as float32, so the reference gets those values: with beta2 = 0.999 in double,
    1 - beta2 differs from the kernel's by 1.3e-5 relative, which shows in exp_avg_sq."""
    out_p, out_m, out_v = [], [], []
    for b in range(p0.shape[0]):
        p = p0[b].double().clone().requires_grad_(True)
        opt = torch.optim.AdamW([p], lr=f32(ens.lr), betas=tuple(f32(x) for x in ens.betas), eps=f32(ens.eps),
                                weight_decay=f32(ens.weight_decay))
        opt.state[p] = {"step": torch.tensor(float(steps[b])), "exp_avg": m0[b].double().clone(),
                        "exp_avg_sq": v0[b].double().clone()}
        p.grad = g[b].double().clone()
        opt.step()
        out_p.append(p.detach()); out_m.append(opt.state[p]["exp_avg"]); out_v.append(opt.state[p]["exp_avg_sq"])
    return torch.stack(out_p), torch.stack(out_m), torch.stack(out_v)


@pytest.mark.parametrize("path", ["step_umma", "step_fp32", "step_layerwise", "adam_step"])
def test_per_object_adamw_state(path):
    """Heterogeneous per-object step numbers and moments. A 1024-float AdamW block spans two rows with different step
    numbers whenever the row pitch is not a multiple of 1024 (hidden 32: 11392)."""
    hidden = 64 if path == "step_layerwise" else 32
    impl = {"step_umma": "umma", "step_fp32": "fp32", "step_layerwise": "layerwise", "adam_step": "umma"}[path]
    B, R, S = len(COUNTERS), 130, 10
    params = vo.init_params(B, hidden, seed=12)
    db = to_dev(vo.synthetic_batch(B, R, S, seed=13))
    ens = make_ensemble(params, 2.0, hidden, impl=impl)
    set_random_state(ens, 14)
    P = ens.count
    p0, m0, v0 = ens.params[:, :P].cpu(), ens.exp_avg[:, :P].cpu(), ens.exp_avg_sq[:, :P].cpu()
    if path == "adam_step":
        g = torch.randn(B, P, generator=torch.Generator().manual_seed(15)) * 0.1
        ens.grads[:, :P] = g.cuda()
        ens.adam_step()
    else:
        # the same state's gradient from a non-fused call (the hidden-32 finisher reduces in the same order)
        probe = make_ensemble(params, 2.0, hidden, impl=impl)
        probe.forward_backward(db)
        g = probe.grads[:, :P].cpu()
        ens.step(db)
    ens.check_status()
    p_ref, m_ref, v_ref = torch_adamw(ens, p0, g, m0, v0, COUNTERS)
    p1, m1, v1 = ens.params[:, :P].cpu().double(), ens.exp_avg[:, :P].cpu().double(), ens.exp_avg_sq[:, :P].cpu().double()
    d_err = max(rel_l2(p1[b] - p0[b].double(), p_ref[b] - p0[b].double()) for b in range(B))
    m_err = max(rel_l2(m1[b], m_ref[b]) for b in range(B))
    v_err = max(rel_l2(v1[b], v_ref[b]) for b in range(B))
    print(f"\n{path}: per-object AdamW vs torch.optim.AdamW (fp64), steps {COUNTERS}")
    assert report("update rel-L2", d_err, BAR_ADAM_DELTA) < BAR_ADAM_DELTA
    assert report("exp_avg rel-L2", m_err, BAR_ADAM_MOM) < BAR_ADAM_MOM
    assert report("exp_avg_sq rel-L2", v_err, BAR_ADAM_MOM) < BAR_ADAM_MOM
    assert ens.step_counter.cpu().tolist() == [c + 1 for c in COUNTERS]
    if path != "step_umma":                               # the fused finisher never touches the grads block
        assert float(ens.grads.abs().sum()) == 0.0
    if ens.image is not None:                             # the fp16 image follows the updated weights
        fresh = ens.image.clone()
        ens.refresh_image()
        assert torch.equal(fresh, ens.image)


# ---- loss-guard granularity ----------------------------------------------------------------------------------------------

GUARD_PATHS = ["step_umma", "step_fp32", "step_layerwise", "split_umma", "fused_adamw"]


def _guard_run(path, params, batch):
    """One optimiser step on ``path``; returns the ensemble."""
    from vmap_b200.lazy import fused_loss
    from vmap_b200.optim import FusedAdamW
    hidden = params["mid1.0.0.weight"].shape[-1]
    impl = {"step_umma": "umma", "step_fp32": "fp32", "step_layerwise": "layerwise"}.get(path, "umma")
    ens = make_ensemble(params, 2.0, hidden, impl=impl)
    before = dict(params=ens.params.clone(), exp_avg=ens.exp_avg.clone(), exp_avg_sq=ens.exp_avg_sq.clone(),
                  image=ens.image.clone())
    if path.startswith("step_"):
        ens.step(batch)
    elif path == "split_umma":                            # the drop-in protocol: backward into grads, AdamW second
        ens.forward_backward(batch)
        ens.adam_step()
    else:                                                 # loss.backward(); optimiser.step() as train.py writes it
        total = torch.zeros(1, device="cuda")
        ens.forward_backward(batch, loss_out=total)
        fused_loss(ens, total).backward()
        FusedAdamW(lr=ens.lr, weight_decay=ens.weight_decay).step()
    torch.cuda.synchronize()
    return ens, before


@pytest.mark.parametrize("path", GUARD_PATHS)
def test_loss_guard_is_per_object(path):
    """Object 1 of three explodes: it keeps its params, moments, fp16 image and step number and its gradient row is
    zeroed; objects 0 and 2 are updated as in a stack without object 1; check_status() raises LossExplode."""
    from vmap_b200.ensemble import LossExplode
    hidden = 64 if path == "step_layerwise" else 32
    B, R, S = 3, 60, 10
    params = vo.init_params(B, hidden, seed=2)
    batch = vo.synthetic_batch(B, R, S, seed=1)
    make_explode(params, batch, 1)
    ens, before = _guard_run(path, params, to_dev(batch))
    assert float(ens.loss_terms[1, 0]) > 1e5
    with pytest.raises(LossExplode):
        ens.check_status()
    for k, v in before.items():
        assert torch.equal(getattr(ens, k)[1], v[1]), k
    assert float(ens.grads[1].abs().sum()) == 0.0
    assert ens.step_counter.cpu().tolist() == [1, 0, 1]
    keep = [0, 2]
    ref, ref_before = _guard_run(path, {k: v[keep] for k, v in params.items()},
                                 to_dev({k: v[keep] for k, v in batch.items()}))
    ref.check_status()
    print(f"\n{path}: objects 0 and 2 against a stack without object 1")
    for name in ("params", "exp_avg", "exp_avg_sq"):
        got, want = getattr(ens, name)[keep], getattr(ref, name)
        if name == "params":
            got, want = got - before["params"][keep], want - ref_before["params"]
        e = max(rel_l2(got[i], want[i]) for i in range(2))
        assert report(f"{name} {'update ' if name == 'params' else ''}rel-L2", e, BAR_GUARD) < BAR_GUARD, name
