"""CPU checks of the fp16-faithful reference of the fused hidden-32 step (oracle/fused_oracle.py).

With every rounding switch off it must be the exact fp64 gradient of oracle.vmap_oracle's model: this validates the
hand-written backward that test_fused_faithful_gpu.py compares the kernel with. With the rounding points moved to the
layer-wise path's places it must equal oracle/lw_oracle.py at hidden 32, so the two restatements differ only where the
kernels do. The saturation regime of the GPU tests is shown to exist here first."""
import pytest
import torch

from oracle import fused_oracle as fo
from oracle import lw_oracle as lw
from oracle import vmap_oracle as vo
from tests._util import rel_l2

SCALE = 2.0
# (B, R, S, label mix, which object has an empty mask)
CASES = [
    dict(B=1, R=7, S=1, empty=None, probs=(0.1, 0.3, 0.6, 0.1)),         # one sample per ray
    dict(B=2, R=9, S=32, empty=None, probs=(0.3, 0.2, 0.5, 0.3)),        # a full warp per ray, mixed labels
    dict(B=3, R=12, S=10, empty="obj", probs=(0.1, 0.3, 0.6, 0.1)),      # object 1 all background: L_d, L_c off
    dict(B=2, R=10, S=14, empty="depth", probs=(0.1, 0.1, 0.2, 0.7)),    # object 0 has no depth rays
]
IDS = ["B{B}R{R}S{S}-{empty}".format(**c) for c in CASES]


def make_batch(c, seed):
    B, R, S = c["B"], c["R"], c["S"]
    if S > 1:
        batch = vo.synthetic_batch(B, R, S, seed=seed, n_cam2surf=min(5, S - 1), empty_prob=c["probs"])
    else:
        batch = vo.synthetic_batch(B, R, 2, seed=seed, n_cam2surf=1, empty_prob=c["probs"])
        batch["pcs"], batch["z"] = batch["pcs"][:, :, :1].contiguous(), batch["z"][:, :, :1].contiguous()
    if c["empty"] == "obj":
        batch["sem"][1] = 0
    elif c["empty"] == "depth":
        batch["mask_depth"][0] = False
    return batch


def exact(params, batch, scale):
    """fp64 autograd through oracle.vmap_oracle."""
    p64 = {k: v.double() for k, v in params.items()}
    b64 = {k: (v.double() if v.is_floating_point() else v) for k, v in batch.items()}
    orc = vo.OracleEnsemble(p64, scale)
    orc.loss(b64).backward()
    g = {k: torch.zeros_like(v) if v.grad is None else v.grad for k, v in orc.params.items()}
    return orc.render(b64), orc.loss_terms(b64), g


def per_object_err(got, ref):
    """Largest rel-L2 over (object, tensor); a reference row that is exactly zero must be matched by zero."""
    worst, where = 0.0, None
    for k in vo.ALL_KEYS:
        g, r = got[k].double().flatten(1), ref[k].double().flatten(1)
        num, den = (g - r).norm(dim=1), r.norm(dim=1)
        e = torch.where(den > 0, num / den.clamp_min(1e-300), num)
        i = int(e.argmax())
        if float(e[i]) >= worst:
            worst, where = float(e[i]), (i, k)
    return worst, where


def same(a, b):
    """Two step results are identical: render, loss terms and every gradient."""
    for x, y in zip(a[0], b[0]):
        assert torch.equal(x, y)
    assert torch.equal(a[1], b[1])
    for k in vo.ALL_KEYS:
        assert torch.equal(a[2][k], b[2][k]), k


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_rounding_off_is_the_exact_gradient(c):
    params = vo.init_params(c["B"], 32, seed=32 + c["R"] + 2)
    batch = make_batch(c, seed=c["S"])
    (d, v, col, o), terms, g_ref = exact(params, batch, SCALE)
    (d1, v1, col1, o1), terms1, g = fo.fused_step(params, SCALE, batch, rounding=fo.ROUND_OFF)
    for a, b in ((d1, d), (v1, v), (col1, col), (o1, o)):
        assert rel_l2(a, b) <= 1e-12
    assert float((terms1 - terms).abs().max()) <= 1e-12 * float(terms.abs().max().clamp_min(1.0))
    e, at = per_object_err(g, g_ref)
    print(f"\n{c}: rounding off vs fp64 autograd {e:.2e} at {at}")
    assert e <= 1e-10, at
    if c["empty"] == "obj":                                    # the whole-batch early-out of L_depth and L_colour
        assert float(terms[:, :2].abs().max()) == 0.0 and float(terms1[:, :2].abs().max()) == 0.0


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_layerwise_placement_is_lw_step(c):
    """Moving each rounding to where the layer-wise path has it gives oracle/lw_oracle.py's step at hidden 32."""
    params = vo.init_params(c["B"], 32, seed=c["R"] + 3)
    batch = make_batch(c, seed=c["S"] + 1)
    r0, t0, g0 = lw.lw_step(params, SCALE, batch)
    r1, t1, g1 = fo.fused_step(params, SCALE, batch, rounding=fo.LW_PLACEMENT)
    for a, b in zip(r1, r0):
        assert rel_l2(a, b) <= 1e-12
    assert float((t1 - t0).abs().max()) <= 1e-12 * float(t0.abs().max().clamp_min(1.0))
    e, at = per_object_err(g1, g0)
    print(f"\n{c}: layer-wise placement vs lw_step {e:.2e} at {at}")
    assert e <= 1e-10, at
    # and the fused placement is a different model: every tensor it rounds differently moves
    _, _, g2 = fo.fused_step(params, SCALE, batch)
    assert per_object_err(g2, g0)[0] > 1e-6


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_own_embedding_signs_and_variance_change_nothing(c):
    params = vo.init_params(c["B"], 32, seed=3)
    batch = make_batch(c, seed=4)
    base = fo.fused_step(params, SCALE, batch)
    e1, e2 = fo.embedding(batch["pcs"], params[vo.PE_KEY], SCALE)
    same(fo.fused_step(params, SCALE, batch, emb=(e1, e2)), base)
    d, _, col, o = base[0]
    same(fo.fused_step(params, SCALE, batch, signs=lw.signs_from_render(d, col, o, batch)), base)
    same(fo.fused_step(params, SCALE, batch, var=base[0][1]), base)


def test_embedding_columns_are_the_oracle_order():
    """fo.embedding with every rounding off is vmap_oracle.unidir_embed (E1 = its first 87 columns, E2 the rest)."""
    batch = make_batch(CASES[1], seed=5)
    dirs = vo.icosahedron_dirs(torch.float64).expand(2, -1, -1) * 1.3
    e1, e2 = fo.embedding(batch["pcs"].double(), dirs, SCALE, fo.ROUND_OFF)
    ref = vo.unidir_embed(batch["pcs"].double(), dirs, torch.full((2,), SCALE, dtype=torch.float64))
    ref = ref.reshape(2, -1, ref.shape[-1])
    assert float((torch.cat([e1, e2], -1) - ref).abs().max()) < 1e-12


def test_fp32_ladder_is_close_to_fp64_cos():
    """The restated fp32 cos ladder stays within a few fp32 ulps x 4^k of fp64 cos (it is a restatement of the
    kernel's arithmetic, not of the exact function)."""
    proj = (torch.rand(1, 4096, 21, generator=torch.Generator().manual_seed(6), dtype=torch.float64) - 0.5) * 40
    proj = proj.float().double()
    c32, c64 = fo.cos_bands(proj, True), fo.cos_bands(proj, False)
    for k in range(6):
        assert float((c32[k] - c64[k]).abs().max()) < 4e-7 * 4.0 ** k, k


def test_counts_override_makes_sub_batches_add_up():
    """A sub-batch run with the full batch's mask counts is that sub-batch's share of the full step."""
    c = CASES[1]
    params = vo.init_params(c["B"], 32, seed=5)
    batch = make_batch(c, seed=6)
    counts = lw.mask_counts(batch["sem"], batch["mask_depth"])
    _, t_full, g_full = fo.fused_step(params, SCALE, batch)
    parts = [fo.fused_step(params, SCALE, {k: v[:, s] for k, v in batch.items()}, counts=counts)
             for s in (slice(0, 4), slice(4, None))]
    assert float((parts[0][1] + parts[1][1] - t_full).abs().max()) < 1e-12
    e, at = per_object_err({k: parts[0][2][k] + parts[1][2][k] for k in vo.ALL_KEYS}, g_full)
    assert e < 1e-12, at


def test_head_gradient_stays_below_fp16_saturation():
    """The regime built to saturate dh16 (one depth ray per object, samples clustered within 1e-3 of the surface, so
    the depth-loss weight 1 / (sqrt(var) + 1e-4) is large) does not reach 65504. dh_a = 10 occ (1 - occ) dL/docc, and
    the depth term's dD/docc shrinks with the same spread of z that makes var small: their product stays bounded, as
    do the opacity (<= 10 LS os / 4 = 6400) and colour (<= 10 LS cs 3 / 4 = 9600) terms at a mask count of one. The
    largest |LS dh| seen here is 1.3e3, a factor 50 below saturation."""
    params = vo.init_params(2, 32, seed=7)
    batch = fo.saturation_batch(2, 64, 10, seed=8)
    aux = {}
    _, _, g = fo.fused_step(params, SCALE, batch, aux=aux)
    top = float(aux["dh"].abs().max())
    print(f"\nhigh-info regime: max |LS dh| = {top:.3e}")
    assert 500.0 < top < fo.HALF_MAX / 8
    assert all(bool(torch.isfinite(v).all()) for v in g.values())
