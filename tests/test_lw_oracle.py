"""CPU checks of the fp16-faithful layer-wise reference (oracle/lw_oracle.py).

With every rounding switch off it must be the exact fp64 gradient of oracle.vmap_oracle's model: this validates the
hand-written backward that the GPU tests (test_layerwise_faithful_gpu.py) compare the kernel with. With the roundings
on it must stay close to the exact gradient: the fp16 stores of the layer-wise path are not what makes its
fp32-oracle bars wide."""
import pytest
import torch

from oracle import lw_oracle as lw
from oracle import vmap_oracle as vo
from tests._util import rel_l2

# (B, R, S, n_cam2surf, label mix, which object has an empty mask)
CASES = [
    dict(B=1, R=7, S=1, empty=None, probs=(0.1, 0.3, 0.6, 0.1)),         # one sample per ray
    dict(B=2, R=9, S=32, empty=None, probs=(0.3, 0.2, 0.5, 0.3)),        # a full warp per ray, more invalid depth
    dict(B=3, R=12, S=10, empty="obj", probs=(0.1, 0.3, 0.6, 0.1)),      # object 1 has no object rays: L_d, L_c off
    dict(B=2, R=10, S=14, empty="depth", probs=(0.1, 0.1, 0.2, 0.7)),    # object 0 has no depth rays; few 'other' labels
]
IDS = ["B{B}R{R}S{S}-{empty}".format(**c) for c in CASES]
HIDDEN = [64, 128, 256]
# Rounding on vs the exact gradient, per (object, tensor) rel-L2, with the exact forward's L1 signs:
# - only the gradient stores (dh16, dYc, dY4..dY1) rounded: worst 5.4e-4 over CASES x HIDDEN, so fp16 underflow of
#   the loss-scaled gradients is small;
# - every rounding on, at 100-300 rays: worst 2.2e-2 (SHAPES_ALL, two seeds each). The forward fp16 stores (embedding,
#   weights, activations) move the gradient far more than the gradient stores do; on 10-ray batches, where bias
#   gradients are sums with heavy cancellation, it reaches 1e-1.
BAR_ROUNDED_DY = 1.5e-3
BAR_ROUNDED_ALL = 5e-2
SHAPES_ALL = [(1, 100, 10, 256), (1, 96, 14, 128), (2, 100, 10, 64), (1, 300, 32, 256)]


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
    g = {k: torch.zeros_like(v) if v.grad is None else v.grad for k, v in orc.params.items()}   # None: not in the loss
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


@pytest.mark.parametrize("H", HIDDEN)
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_rounding_off_is_the_exact_gradient(c, H):
    params = vo.init_params(c["B"], H, seed=H + c["R"] + 2)
    batch = make_batch(c, seed=c["S"])
    (d, v, col, o), terms, g_ref = exact(params, batch, 5.0)
    (d1, v1, col1, o1), terms1, g = lw.lw_step(params, 5.0, batch, rounding=lw.ROUND_OFF)
    for a, b in ((d1, d), (v1, v), (col1, col), (o1, o)):
        assert rel_l2(a, b) <= 1e-12
    assert float((terms1 - terms).abs().max()) <= 1e-12 * float(terms.abs().max().clamp_min(1.0))
    e, at = per_object_err(g, g_ref)
    print(f"\nH={H} {c}: rounding off vs fp64 autograd {e:.2e} at {at}")
    assert e <= 1e-10, at
    if c["empty"] == "obj":                                    # the whole-batch early-out of L_depth and L_colour
        assert float(terms[:, :2].abs().max()) == 0.0 and float(terms1[:, :2].abs().max()) == 0.0


def rounded_vs_exact(params, batch, rounding):
    """Per-object error of a rounded step against the exact one, both with the exact forward's L1 signs (so a ray
    whose residual sits within the fp16 noise does not flip)."""
    (d, _, col, o), _, g_ref = lw.lw_step(params, 5.0, batch, rounding=lw.ROUND_OFF)
    signs = lw.signs_from_render(d, col, o, batch)
    _, _, g = lw.lw_step(params, 5.0, batch, signs=signs, rounding=rounding)
    return per_object_err(g, g_ref)


@pytest.mark.parametrize("H", HIDDEN)
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_rounded_gradient_stores_stay_near_the_exact_gradient(c, H):
    params = vo.init_params(c["B"], H, seed=H + c["R"] + 2)
    e, at = rounded_vs_exact(params, make_batch(c, seed=c["S"]), lw.Rounding(emb=False, weights=False, acts=False))
    print(f"\nH={H} {c}: dY stores rounded {e:.2e} at {at} (bar {BAR_ROUNDED_DY:.1e})")
    assert e < BAR_ROUNDED_DY, at


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("B,R,S,H", SHAPES_ALL)
def test_all_roundings_stay_near_the_exact_gradient(B, R, S, H, seed):
    params = vo.init_params(B, H, seed=seed)
    e, at = rounded_vs_exact(params, vo.synthetic_batch(B, R, S, seed=seed + 10, n_cam2surf=5), lw.ROUND_ALL)
    print(f"\n{B}x{R}x{S} H={H}: all roundings {e:.2e} at {at} (bar {BAR_ROUNDED_ALL:.0e})")
    assert e < BAR_ROUNDED_ALL, at


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_sign_override_with_own_signs_changes_nothing(c):
    params = vo.init_params(c["B"], 128, seed=3)
    batch = make_batch(c, seed=4)
    (d, _, col, o), terms, g = lw.lw_step(params, 5.0, batch)
    _, terms1, g1 = lw.lw_step(params, 5.0, batch, signs=lw.signs_from_render(d, col, o, batch))
    assert torch.equal(terms, terms1)
    for k in vo.ALL_KEYS:
        assert torch.equal(g[k], g1[k]), k


def test_counts_override_makes_sub_batches_add_up():
    """A sub-batch run with the full batch's mask counts is that sub-batch's share of the full step."""
    c = CASES[1]
    params = vo.init_params(c["B"], 64, seed=5)
    batch = make_batch(c, seed=6)
    counts = lw.mask_counts(batch["sem"], batch["mask_depth"])
    _, t_full, g_full = lw.lw_step(params, 5.0, batch)
    parts = [lw.lw_step(params, 5.0, {k: v[:, s] for k, v in batch.items()}, counts=counts)
             for s in (slice(0, 4), slice(4, None))]
    assert float((parts[0][1] + parts[1][1] - t_full).abs().max()) < 1e-12
    e, at = per_object_err({k: parts[0][2][k] + parts[1][2][k] for k in vo.ALL_KEYS}, g_full)
    assert e < 1e-12, at
