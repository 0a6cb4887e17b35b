"""The fused hidden-32 step (impl="umma") against an fp16-faithful reference that reads the kernel's own embedding, at
per-object bars.

test_umma_gpu.py compares this kernel with the fp32 oracle at a gradient rel-L2 of 4e-2, and
test_fused_invariants_gpu.py with itself, which cannot see an error every arrangement of the rays shares (a misplaced
fp16 rounding, a wrong loss scale). oracle/fused_oracle.py rounds where the kernel rounds. The one input it cannot
restate closely enough is the embedding: the kernel's sin bands come from a MUFU sin / cos pair and an angle-doubling
ladder, and their fp16 values differ from fp16 of fp64 sin (test_pe_accuracy_against_fp64 measures by how much). So
``probe_embedding`` reads the kernel's own fp16 embedding back through ``eval_points``, which runs the same E0 code:
129 probe objects per real object, each with selector weights that turn one embedding column into its output
exactly. The reference then starts from the kernel's embedding, takes the L1 signs from the kernel's render, and what
is left between the two is fp32 accumulation order against fp64 and the fp16 roundings it moves.

Run with -s to see every measured value next to its bar.
"""
import pytest
import torch

from oracle import fused_oracle as fo
from oracle import vmap_oracle as vo
from tests._util import make_ensemble, to_dev

pytestmark = pytest.mark.gpu

# Bars: about four to five times the worst value measured over SEEDS on an H100 80GB HBM3 at a 700 W power limit.
# Per (object, tensor) gradient rel-L2 against the faithful reference. What is left is fp32 accumulation order against
# fp64, and the fp16 activation / relu-gate flips it causes; on an object of a few hundred points one flip can
# dominate a tensor, so, as in test_layerwise_faithful_gpu.py, the bar depends on the point count:
BAR_GRAD = 3e-3         # >= 8,192 points per object: worst 5.3e-4
BAR_GRAD_SMALL = 5e-2   # fewer: worst 1.1e-2 (160 x 60 x 10, one object's color_linear.0.weight); typical 1e-4
BAR_RENDER = 2e-3       # per (object, output) rel-L2 of depth, var, colour, opacity, >= 8,192 points: worst 4.5e-4
BAR_RENDER_SMALL = 1.5e-2   # fewer: worst 3.0e-3 (2,700 objects of one 2-sample ray: one flip is the whole object)
BAR_LOSS = 1.2e-3       # per (object, term) relative loss-term difference: worst 2.7e-4 (65,536 rays: fp32 sums)
BAR_EVAL = 1.5e-4       # eval_points: per object rel-L2 of raw alpha and of colour: worst 3.6e-5
BAR_EXACT = 2.5e-2      # kernel against the exact fp64 model (rounding off, the kernel's signs): worst 5.7e-3
# PE accuracy against fp16(fp64 sin) of the same fp32 projection, per band k = 0..5. The worst absolute error is one
# fp16 ulp at |sin| >= 0.5 (2^-11 = 4.9e-4) in every band; in ulps the worst distance grows with k as the ladder
# doubles the seed error near sin = 0, where fp16 ulps are finest: 4, 7, 23, 46, 140, 351 ulps for k = 0..5.
# Direction 20 (sin_ladder) is no worse than the rest (k = 5: 205 ulps).
BAR_PE_ABS = 2e-3
BAR_PE_ULP = [16, 32, 96, 192, 600, 1500]
SEEDS = [41, 42, 43]
SCALE = 2.0


# ---- probe: the kernel's own fp16 embedding ---------------------------------------------------------------------------

E1, E2 = vo.emb_sizes()
N_PROBE = E1 + E2                       # 129: one probe object per embedding column
CH_SCALE = (1.0, 2.0 ** 7, 2.0 ** 14)   # colour-channel gains of the probes (powers of two: exact in fp16)
_probe_cache = {}


def probe_params(dirs):
    """[129, *shape] fp32 probe weights for one real object's PE directions ``dirs`` [21, 3]. Probe j < 87 routes emb1
    column j as +e / -e through fc1..fc4 (identity layers, zero biases): raw alpha = 10 (relu(e) - relu(-e)) = 10 e,
    every accumulation has one nonzero term, and the same pair reaches hc[0], hc[1] and the colour head. Probe 87 + j2
    routes emb2 column j2 into hc[0], hc[1] only (fc4 = 0). Colour channel c returns sigmoid(CH_SCALE[c] e)."""
    shapes = vo.param_shapes(32)
    p = {k: torch.zeros((N_PROBE,) + s) for k, s in shapes.items()}
    eye = torch.eye(32)
    ar = torch.arange(E1)
    p["in_layer.0.weight"][ar, 0, ar] = 1.0
    p["in_layer.0.weight"][ar, 1, ar] = -1.0
    p["mid1.0.0.weight"][:] = eye
    p["cat_layer.0.weight"][:, :, :32] = eye
    p["mid2.0.0.weight"][:] = eye
    p["out_alpha.weight"][:, 0, 0], p["out_alpha.weight"][:, 0, 1] = 1.0, -1.0
    p["color_linear.0.weight"][:E1, :, :32] = eye
    a2 = torch.arange(E2)
    p["color_linear.0.weight"][E1 + a2, 0, 32 + a2] = 1.0
    p["color_linear.0.weight"][E1 + a2, 1, 32 + a2] = -1.0
    for c, s in enumerate(CH_SCALE):
        p["out_color.weight"][:, c, 0], p["out_color.weight"][:, c, 1] = s, -s
    p[vo.PE_KEY][:] = dirs.float().cpu()
    return p


def _probe_ensemble(n):
    if n not in _probe_cache:
        _probe_cache.clear()
        _probe_cache[n] = make_ensemble(vo.init_params(n, 32, seed=0), SCALE, 32, impl="umma")
    return _probe_cache[n]


def _recover_colour(col):
    """col [..., 3] fp32 sigmoid(CH_SCALE[c] e) -> (e rounded to fp16, where it could be read): invert the most
    amplified channel whose sigmoid is still well conditioned (|x| <= 6), then check that e re-encodes to all three
    outputs. Only a t column far outside the scene saturates channel 0."""
    y = col.double().clamp(1e-30, 1 - 1e-16)
    x = torch.log(y) - torch.log1p(-y)
    sc = torch.tensor(CH_SCALE, dtype=torch.float64, device=col.device)
    ok = x.abs() <= 6.0
    c = (ok * torch.arange(1, 4, device=col.device)).argmax(-1, keepdim=True)     # last well-conditioned channel
    e = (x.gather(-1, c) / sc[c]).squeeze(-1).half().double()
    valid = ok[..., 0]
    err = ((torch.sigmoid(e[..., None] * sc) - col.double()).abs().amax(-1) * valid).max()
    assert float(err) < 1e-6, f"probe: recovered embedding does not re-encode (err {float(err):.2e})"
    return e, valid


def probe_embedding(params, scale, points):
    """The kernel's fp16 embedding of ``points`` [B,N,3] for the real objects ``params``: (E1 [B,N,87],
    E2 [B,N,42]) in fp64, reference column order. Checks that every emb1 column read through the colour path equals
    its exact alpha-path value and that every recovered value re-encodes to the kernel's outputs."""
    B, N, _ = points.shape
    m = max(1, min(B, 4096 // N_PROBE, (1 << 25) // (N_PROBE * N)))
    e1s, e2s = [], []
    sc = torch.as_tensor(scale, dtype=torch.float32).expand(B)
    for b0 in range(0, B, m):
        bs = list(range(b0, min(B, b0 + m)))
        ens = _probe_ensemble(len(bs) * N_PROBE)
        pp = [probe_params(params[vo.PE_KEY][b]) for b in bs]
        ens.load_stacked({k: torch.cat([q[k] for q in pp]) for k in vo.ALL_KEYS})
        ens.scale.copy_(sc[bs].repeat_interleave(N_PROBE))
        pts = points[bs].repeat_interleave(N_PROBE, 0).contiguous()
        alpha, col = ens.eval_points(pts)
        alpha = alpha.view(len(bs), N_PROBE, N).double()
        col = col.view(len(bs), N_PROBE, N, 3)
        e1 = alpha[:, :E1] / 10.0
        assert torch.equal(e1.half().double(), e1), "probe: alpha path is not an fp16 value x 10"
        e_col, valid = _recover_colour(col)
        assert bool(valid[:, E1:].all()), "probe: an emb2 value saturated colour channel 0"
        assert bool(valid[:, 3:E1].all()), "probe: an emb1 sin value saturated colour channel 0"
        assert torch.equal(torch.where(valid[:, :E1], e_col[:, :E1], e1), e1), \
            "probe: colour path disagrees with the alpha path"
        e1s.append(e1.transpose(1, 2))
        e2s.append(e_col[:, E1:].transpose(1, 2))
    return torch.cat(e1s), torch.cat(e2s)


# ---- helpers -----------------------------------------------------------------------------------------------------------

def make_batch(B, R, S, seed):
    return fo.synthetic(B, R, S, seed)


def grads_of(ens, batch, counts=None):
    ens.grads.zero_()
    ens.forward_backward(batch, counts=counts)
    return ens.stacked(ens.grads.clone()), ens.loss_terms.clone()


def grad_err(got, ref):
    """Largest relative L2 error over (object, tensor) pairs of two {key: [B, *shape]} gradients, and where it is."""
    worst, where = 0.0, None
    for k in vo.ALL_KEYS:
        g, r = got[k].double().flatten(1), ref[k].double().flatten(1).to(got[k].device)
        num, den = (g - r).norm(dim=1), r.norm(dim=1)
        e = torch.where(den > 0, num / den.clamp_min(1e-300), num)        # an exactly-zero row must stay zero
        i = int(e.argmax())
        if float(e[i]) > worst or where is None:
            worst, where = float(e[i]), (i, k)
    return worst, where


def loss_err(got, ref):
    """Per (object, term) relative difference; terms below 1e-3 are compared absolutely (the opacity residual
    |O - 1| of an opaque object is a cancellation in the kernel's fp32 sum)."""
    got, ref = got.double(), ref.double().to(got.device)
    return float(((got - ref).abs() / ref.abs().clamp_min(1e-3)).max())


def render_err(got, ref, z):
    """Per (object, output) rel-L2 of depth, var, colour and opacity. The variance error is taken relative to the
    rays' largest z squared: the kernel's fp32 sum of w (z - D)^2 cancels to an absolute error on that scale."""
    worst = 0.0
    zz = z.double().amax(-1) ** 2
    for i, (g, r) in enumerate(zip(got, ref)):
        g, r = g.double().flatten(1), r.double().flatten(1).to(g.device)
        den = zz.norm(dim=1) if i == 1 else r.norm(dim=1)
        worst = max(worst, float(((g - r).norm(dim=1) / den.clamp_min(1e-30)).max()))
    return worst


def report(name, value, bar):
    print(f"  {name}: {value:.3e} (bar {bar:.1e})")
    return value


def reference(params, db, render, counts=None, emb=None, rounding=fo.ROUND_ALL, ls=fo.LS, aux=None):
    """The faithful reference in fp64 on the GPU, with the kernel's L1 signs and ray variances and (default) its probed
    embedding."""
    d, v, c, o = render
    dev = {k: v.cuda() for k, v in params.items()}
    if emb is None:
        B, R, S, _ = db["pcs"].shape
        emb = probe_embedding(params, SCALE, db["pcs"].reshape(B, R * S, 3))
    return fo.fused_step(dev, SCALE, db, counts=counts, signs=fo.signs_from_render(d, c, o, db), emb=emb,
                         var=v, rounding=rounding, ls=ls, aux=aux)


def check(ens, params, db, counts=None, label=""):
    """Kernel against the reference: render, loss terms, gradient. Returns (grad error, kernel grads, reference)."""
    render = ens.render(db)
    g, lt = grads_of(ens, db, counts)
    ref = reference(params, db, render, counts)
    ge, at = grad_err(g, ref[2])
    print(f"\n{label}: worst gradient at {at}")
    B, R, S, _ = db["pcs"].shape
    bar, r_bar = (BAR_GRAD, BAR_RENDER) if R * S >= 8192 else (BAR_GRAD_SMALL, BAR_RENDER_SMALL)
    assert report("render", render_err(render, ref[0], db["z"]), r_bar) < r_bar
    assert report("loss terms", loss_err(lt, ref[1]), BAR_LOSS) < BAR_LOSS
    assert report("grad", ge, bar) < bar, at
    return ge, g, ref


# ---- PE accuracy --------------------------------------------------------------------------------------------------------

def _ulps(a, b):
    """Distance in fp16 ulps between fp16-valued fp64 tensors (ordered integer view of the bit patterns)."""
    def ordered(x):
        i = x.half().view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (ordered(a) - ordered(b)).abs()


def pe_points(seed):
    """Points for the PE check, in units of the scale: the scene range, |proj| up to 64, projections at and next to
    integers and half-integers on the axis directions (3 = x, 9 = y, 17 = z), and negatives."""
    g = torch.Generator().manual_seed(seed)
    scene = (torch.rand(20000, 3, generator=g) - 0.5) * 2.0
    far = (torch.rand(4000, 3, generator=g) - 0.5) * 128.0
    base = torch.randint(-40, 41, (6000, 1), generator=g).float() * 0.5
    eps = torch.tensor([0.0, 2.0 ** -23, -2.0 ** -23, 2.0 ** -20, -2.0 ** -20, 2.0 ** -12, -2.0 ** -12, 1e-3])
    tie = base + eps[torch.randint(0, len(eps), (6000, 1), generator=g)] * base.abs().clamp_min(1.0)
    ax = torch.zeros(6000, 3)
    col = torch.randint(0, 3, (6000,), generator=g)
    ax[torch.arange(6000), col] = tie[:, 0]
    return torch.cat([scene, far, ax]) * SCALE


@pytest.mark.parametrize("seed", SEEDS)
def test_pe_accuracy_against_fp64(seed):
    """The kernel's fp16 sin bands (MUFU sin / cos of the reduced angle, then angle doubling in fp32) against fp16 of
    fp64 sin of the same fp32 projection, per band k: max absolute error and max ulp distance. The t columns must be
    exact. Direction 20 (the separate sin_ladder) is reported on its own."""
    params = vo.init_params(1, 32, seed=seed)
    pts = pe_points(seed)[None].cuda()
    e1, e2 = probe_embedding(params, SCALE, pts)
    r1, r2 = fo.embedding(pts[:, :, None], params[vo.PE_KEY].double().cuda(), SCALE)
    assert torch.equal(e1[..., :3], r1[..., :3]), "t columns"
    got = torch.cat([e1[..., 3:], e2], -1).view(-1, 6, 21)
    ref = torch.cat([r1[..., 3:], r2], -1).view(-1, 6, 21)
    print(f"\nseed {seed}: {pts.shape[1]} points, kernel sin bands vs fp16(fp64 sin)")
    for k in range(6):
        ab = float((got[:, k] - ref[:, k]).abs().max())
        u = _ulps(got[:, k], ref[:, k])
        u20 = int(u[:, 20].max())
        frac = float((u > 0).double().mean())
        print(f"  k={k}: max |err| {ab:.3e}, max ulps {int(u.max())} (dir 20: {u20}), "
              f"fraction not bit-equal {frac:.3e} (bars {BAR_PE_ABS:.0e}, {BAR_PE_ULP[k]} ulps)")
        assert ab <= BAR_PE_ABS, k
        assert BAR_PE_ULP[k] is None or int(u.max()) <= BAR_PE_ULP[k], k


# ---- parity on the shape grid -------------------------------------------------------------------------------------------

# (B, R, S): the invariants test's SHAPES, every SC instantiation (S = 10, 14 and the generic kernel), R below one tile,
# exactly one tile pair, an odd tile count, BASELINE cfg 3's object count, and a run near MAX_OBJ_SMEM (2773 objects)
GRID = [(4, 301, 10), (5, 30, 10), (2, 100, 14), (1, 64, 16), (3, 40, 1), (2, 33, 20), (2, 50, 32), (20, 1200, 10),
        (2, 50, 2), (2, 50, 3), (2, 40, 31),
        (2, 5, 10), (2, 24, 10), (2, 60, 10),
        (160, 60, 10), (2700, 1, 2)]
GRID_IDS = ["B{}R{}S{}".format(*c) for c in GRID]


def setup(B, R, S, seed):
    params = vo.init_params(B, 32, seed=seed)
    return params, to_dev(make_batch(B, R, S, seed + 100)), make_ensemble(params, SCALE, 32, impl="umma")


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("cfg", GRID, ids=GRID_IDS)
def test_faithful_parity(cfg, seed):
    params, db, ens = setup(*cfg, seed)
    check(ens, params, db, label=f"{cfg} seed {seed}")


# ---- edges ----------------------------------------------------------------------------------------------------------------

def rays(batch, sl):
    return {k: v[:, sl] for k, v in batch.items()}


@pytest.mark.parametrize("case", ["unaligned_rows", "counts_in", "empty_object"])
def test_edges(case):
    """Label / mask rows that are not 4-byte aligned (an odd ray count and a slice starting at ray 1: the scalar count
    loop), mask counts supplied from outside, and an object without object rays (the any-empty early-out turns
    L_depth and L_colour off for every object)."""
    params, db, ens = setup(5, 131, 10, 44)
    counts = None
    if case == "unaligned_rows":
        db = rays(db, slice(1, 131))
    elif case == "counts_in":
        full = db
        db = rays(db, slice(3, 100))
        counts = ens.mask_counts(full)
    else:
        db["sem"][2] = 0
    check(ens, params, db, counts=counts, label=case)
    if case == "empty_object":
        assert float(ens.loss_terms[:, :2].abs().max()) == 0.0


def exact_distance(params, db, render, g_kernel, aux_label):
    """Kernel and faithful reference against the exact fp64 model (every rounding off, the kernel's L1 signs)."""
    d, var, c, o = render
    dev = {k: v.cuda() for k, v in params.items()}
    _, _, g_exact = fo.fused_step(dev, SCALE, db, signs=fo.signs_from_render(d, c, o, db), var=var,
                                  rounding=fo.ROUND_OFF)
    e_k, at = grad_err(g_kernel, g_exact)
    print(f"  {aux_label}: kernel vs exact fp64 model {e_k:.3e} at {at}")
    return e_k, g_exact


@pytest.mark.parametrize("regime", ["high_info", "underflow"])
def test_regimes(regime):
    """high_info: one depth ray per object and samples within 1e-3 of the surface, the largest loss-scaled head
    gradient the losses produce (it stays far below fp16 saturation, see test_fused_oracle.py). underflow: 65,536 rays
    per object, so the 1 / count loss weights push much of the loss-scaled dY into fp16 subnormals or to zero."""
    if regime == "high_info":
        B, R, S = 2, 64, 10
        batch = fo.saturation_batch(B, R, S, seed=45)
    else:
        B, R, S = 1, 65536, 10
        batch = make_batch(B, R, S, 46)
    params = vo.init_params(B, 32, seed=47)
    db = to_dev(batch)
    ens = make_ensemble(params, SCALE, 32, impl="umma")
    ge, g, ref = check(ens, params, db, label=regime)
    aux = {}
    reference(params, db, ens.render(db), aux=aux)
    dh = aux["dh"]
    nz = dh != 0
    sub = (dh.abs() < 2.0 ** -14) & nz
    zero16 = (dh.abs() < 2.0 ** -25) & nz
    print(f"  max |LS dh| {float(dh.abs().max()):.3e}; of the nonzero dh: {float(sub.double().sum() / nz.sum()):.3e} "
          f"subnormal in fp16, {float(zero16.double().sum() / nz.sum()):.3e} flush to zero")
    e_k, _ = exact_distance(params, db, ens.render(db), g, regime)
    assert report("kernel vs exact fp64 model", e_k, BAR_EXACT) < BAR_EXACT


# ---- eval_points --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N", [1, 127, 128, 129, 70001])
def test_eval_points_forward(N):
    """Raw alpha (x10) and sigmoid colour of eval_points at hidden 32 against the faithful forward on the kernel's
    embedding, per object."""
    B = 3
    params = vo.init_params(B, 32, seed=48)
    ens = make_ensemble(params, SCALE, 32, impl="umma")
    pts = ((torch.rand(B, N, 3, generator=torch.Generator().manual_seed(N)) - 0.5) * 4.0).cuda()
    a, c = ens.eval_points(pts)
    emb = probe_embedding(params, SCALE, pts)
    ra, rc = fo.fused_forward({k: v.cuda() for k, v in params.items()}, SCALE, pts, emb=emb)
    ea = float(((a.double() - ra).norm(dim=1) / ra.norm(dim=1)).max())
    ec = float(((c.double() - rc).flatten(1).norm(dim=1) / rc.flatten(1).norm(dim=1)).max())
    print(f"\nN={N}")
    assert report("raw alpha", ea, BAR_EVAL) < BAR_EVAL
    assert report("colour", ec, BAR_EVAL) < BAR_EVAL


# ---- power ----------------------------------------------------------------------------------------------------------------

POWER_CASES = [("cfg2", (20, 1200, 10)), ("high_info", None), ("underflow", None)]


def _power_setup(name, shape):
    if name == "cfg2":
        params, db, ens = setup(*shape, 41)
    elif name == "high_info":
        params = vo.init_params(2, 32, seed=47)
        db = to_dev(fo.saturation_batch(2, 64, 10, seed=45))
        ens = make_ensemble(params, SCALE, 32, impl="umma")
    else:
        params = vo.init_params(1, 32, seed=47)
        db = to_dev(make_batch(1, 65536, 10, 46))
        ens = make_ensemble(params, SCALE, 32, impl="umma")
    return params, db, ens


@pytest.mark.parametrize("name,shape", POWER_CASES, ids=[c[0] for c in POWER_CASES])
def test_rounding_switches_are_resolved(name, shape):
    """Each rounding switch flipped on its own (and the loss scale halved to 2^7): wherever the flip moves the
    reference by more than 3x the gradient bar, the kernel must fail the bar against the flipped reference. The flips
    below the comparator's resolution are printed as such. Measured at cfg 2 (20 x 1200 x 10): the fp16 weight image
    (3.2e-2) and the fp16 activations (2.5e-2) are resolved; the head weights' fp16 image (3.0e-3) sits at the bar;
    emb (exact fp64 sin instead of fp16: 0 once the kernel's embedding is given), proj32, dh, dh_feeds, dyc, dgrad,
    cos32, dproj, t16 and the loss scale 2^7 move the reference by 5e-6 .. 5e-4, below the comparator's resolution.
    The high-info and underflow regimes resolve only the weight image."""
    params, db, ens = _power_setup(name, shape)
    render = ens.render(db)
    g, _ = grads_of(ens, db)
    B, R, S, _ = db["pcs"].shape
    emb = probe_embedding(params, SCALE, db["pcs"].reshape(B, R * S, 3))
    _, _, g_ref = reference(params, db, render, emb=emb)
    base, _ = grad_err(g, g_ref)
    print(f"\n{name}: kernel vs reference {base:.3e} (bar {BAR_GRAD:.1e})")
    flips = [(s, fo.flipped(s), fo.LS) for s in fo.SWITCHES] + [("ls=2^7", fo.ROUND_ALL, 128.0)]
    for label, rnd, ls in flips:
        _, _, g_flip = reference(params, db, render, emb=None if label in ("emb",) else emb, rounding=rnd, ls=ls)
        moved, _ = grad_err(g_flip, g_ref)
        e_k, at = grad_err(g, g_flip)
        verdict = "resolved" if moved > 3 * BAR_GRAD else "below resolution"
        print(f"  {label:>8}: reference moves {moved:.3e}; kernel vs flipped {e_k:.3e} at {at} ({verdict})")
        if moved > 3 * BAR_GRAD:
            assert e_k > BAR_GRAD, label


def test_dropped_tile_is_rejected():
    """BASELINE cfg 2: the gradient minus one tile of object 1 (a sub-batch run with the full counts) fails the
    reference's gradient bar, which the fp32-oracle bars cannot do (test_fused_invariants_gpu.py)."""
    params, db, ens = setup(20, 1200, 10, 41)
    nr = 4 * (32 // 10)
    counts = ens.mask_counts(db)
    render = ens.render(db)
    g_full, _ = grads_of(ens, db)
    g_tile, _ = grads_of(ens, rays(db, slice(3 * nr, 4 * nr)), counts=counts)
    g_bad = {k: v.clone() for k, v in g_full.items()}
    for k in vo.ALL_KEYS:
        g_bad[k][1] -= g_tile[k][1]
    _, _, g_ref = reference(params, db, render)
    ok, _ = grad_err(g_full, g_ref)
    bad, at = grad_err(g_bad, g_ref)
    print(f"\ntile 3 of object 1 dropped: intact {ok:.3e}, dropped {bad:.3e} at {at}")
    report("dropped (must FAIL the bar by 3x)", bad, BAR_GRAD)
    assert ok < BAR_GRAD and bad > 3 * BAR_GRAD
