"""CPU: the host restatement of the sampler's Philox draws (oracle/philox_oracle.py).

Known-answer vectors pin the generator, the counter-layout checks pin that no two draws of a launch share a
counter, and the statistics of the restated scheme (10^6-10^7 draws, fixed seeds) are the evidence that the scheme
is distributionally right.  The power test shows why the GPU comparison has to be exact: deliberately wrong draw
schemes pass every range / ordering check of the Philox-mode GPU test."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import philox_oracle as po
from oracle import sampler_oracle as so
from tests._util import GOLDEN


# ---- the generator ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answer_vectors(ctr, key, want):
    """Random123's known-answer vectors for Philox4x32-10."""
    got = po.philox4x32_10(*ctr, *key)
    assert tuple(int(x) for x in got) == want
    # vectorised: the same counter in a batch of others gives the same words
    c0 = np.array([1, ctr[0], 7], np.uint64)
    assert tuple(int(x[1]) for x in po.philox4x32_10(c0, *ctr[1:], *key)) == want


def test_u01_and_seed_key():
    assert po.u01(np.uint32(0)) == 0 and po.u01(np.uint32(0xFFFFFFFF)) == np.float32(1 - 2.0 ** -24)
    assert po.u01(np.uint32(0xFF000001)) == np.float32(2.0 ** -24)          # only the low 24 bits count
    assert po.seed_key(2 ** 32 + 5) == (5, 1) and po.seed_key(2 ** 63 - 1) == (0xFFFFFFFF, 0x7FFFFFFF)


# ---- counter layout --------------------------------------------------------------------------------------------------
def _packed(c):
    return c[:, 0].astype(np.uint64) | (c[:, 1].astype(np.uint64) << np.uint64(32))


def test_counters_of_a_launch_are_distinct():
    """B = 1024 objects x N = 4800 rays at S = 32 (n1 = n2 = 16), at two consecutive offsets.  Object b's counters are
    (c0, c1, b, offset): words c2 / c3 separate objects and offsets, so the launch's counters are distinct exactly
    when one object's (c0, c1) pairs are -- checked directly, with the c2 / c3 words checked at both ends of the
    object range."""
    B, F, P, n1, n2 = 1024, 100, 48, 16, 16
    off = 2 ** 31 + 7
    base = po.sampler_counters(0, off, F, P, n1, n2)
    pairs = _packed(base)
    assert np.unique(pairs).size == pairs.size
    assert len(base) == F + F * P * (1 + 8 + 4)
    for o in (off, off + 1):
        for b in (0, 1, B - 2, B - 1):
            c = po.sampler_counters(b, o, F, P, n1, n2)
            assert np.array_equal(_packed(c), pairs) and (c[:, 2] == b).all() and (c[:, 3] == o).all()
    # the offset word is the low 32 bits: offsets 2^32 apart draw the same counters
    assert np.array_equal(po.sampler_counters(3, 5, 2, 3, 1, 9), po.sampler_counters(3, 5 + 2 ** 32, 2, 3, 1, 9))


def test_counter_layout_limits():
    """c0 = i * 8 + chunk: distinct while the chunk index stays below 8 (S <= 32) and i * 8 + 7 < 2^32 (N < 2^29)."""
    assert (2 ** 29 - 1) * 8 + 7 == 2 ** 32 - 1                    # the last ray of the largest launch still fits
    assert (32 + 3) // 4 == 8 and (33 + 3) // 4 == 9               # S = 33 would need chunk 8 == chunk 0 of ray i+1
    c = po.sampler_counters(0, 0, 1, 2, 16, 16)
    assert c[:, 0].max() == 1 * 8 + 7


def test_surface_sampler_counters_and_the_one_overlap():
    """The two layouts side by side: the surface sampler's counter (i, i >> 32, 4, 0) is the ray sampler's stream 0
    (keyframe draws) of object 4 at offset 0.  With equal seeds the two share those draws; the uses are unrelated."""
    n = 4096
    surf = set(map(tuple, po.surface_counters(n).tolist()))
    for b, off in ((4, 0), (4, 1), (3, 0), (5, 0)):
        ray = po.sampler_counters(b, off, 64, 8, 5, 9)
        common = [r for r in map(tuple, ray.tolist()) if r in surf]
        if (b, off) == (4, 0):
            assert len(common) == 64 and all(r[1] == po.STREAM_KF for r in common)
        else:
            assert not common
    c = po.surface_counters(3)
    assert c.tolist() == [[0, 0, 4, 0], [1, 0, 4, 0], [2, 0, 4, 0]]


def test_surface_uniforms_layout():
    u = po.surface_uniforms(123, 1000)
    assert u.shape == (1000, 3) and (u >= 0).all() and (u < 1).all()
    k0, k1 = po.seed_key(123)
    o = po.philox4x32_10(999, 0, 4, 0, k0, k1)
    assert u[999, 1] == int(o[2]) / 2 ** 32 and u[999, 2] == int(o[3]) / 2 ** 32
    assert u[999, 0] == ((int(o[0]) >> 5) * 2 ** 26 + (int(o[1]) >> 6)) / 2 ** 53


# ---- the keyframe rule -----------------------------------------------------------------------------------------------
def test_keyframe_rule_at_the_edges():
    """n_kf > 2: the last two draws are the latest keyframes; n_frames == 1 takes latest[1] (the reference raises
    there: torch.randint of a negative size); n_kf <= 2 draws every frame."""
    kf = po.keyframe_draws(9, 0, 0, 12, 7, [2, 0])
    assert kf[-2:].tolist() == [2, 0] and (kf[:-2] < 7).all() and (kf >= 0).all()
    assert po.keyframe_draws(9, 0, 0, 1, 5, [3, 1]).tolist() == [1]
    assert po.keyframe_draws(9, 0, 0, 2, 3, [2, 0]).tolist() == [2, 0]
    k2 = po.keyframe_draws(9, 0, 0, 400, 2, [1, 0])
    assert set(k2.tolist()) == {0, 1}
    with pytest.raises(RuntimeError):
        so.draw_randoms_reference_order(None, 5, [3, 1], 1, 4, torch.zeros(5, 4), torch.zeros(5, 8, 8, 4),
                                        torch.zeros(5, 8, 8), so.SamplerCfg())


def test_pixel_indices_clamp_to_the_image():
    """A box reaching past the image: the CUDA sampler clamps the pixel, and so does the restatement when given the
    image size.  Unclamped, the high side would index out of range and the low side (negative) would wrap to the
    opposite edge under torch indexing."""
    bbox = torch.tensor([[-3.5, 12.5, -1.0, 9.25]])
    u = torch.tensor([[0.0, 0.1, 0.5, 0.99, 1 - 2.0 ** -24]])
    iw, ih = so.pixel_indices(torch.zeros(1, dtype=torch.long), u, u, bbox, wh=(10, 8))
    assert iw.tolist() == [[0, 0, 4, 9, 9]] and ih.tolist() == [[0, 0, 4, 7, 7]]
    iw0, _ = so.pixel_indices(torch.zeros(1, dtype=torch.long), u, u, bbox)
    assert iw0.max() == 12 and iw0.min() == -3


# ---- statistics of the scheme ----------------------------------------------------------------------------------------
P_MIN = 1e-3          # fixed seeds: every p-value below is a fixed number, far above this


@pytest.mark.parametrize("n_kf", [3, 5, 7])
def test_keyframe_draws_are_uniform(n_kf):
    n = 10 ** 6
    kf = np.concatenate([po.keyframe_draws(17, off, b, n // 4 + 2, n_kf, [0, 0])[:-2] for b, off in
                         ((0, 0), (1, 0), (0, 1), (900, 2 ** 31 + 7))])
    counts = np.bincount(kf, minlength=n_kf)
    assert counts.size == n_kf
    assert stats.chisquare(counts).pvalue > P_MIN


def test_pixels_are_uniform_inside_a_fractional_box():
    """Columns / rows of a fractional box [3.3, 17.8) x [0.6, 9.1): integer k is drawn with probability
    |[k, k+1) n [lo, hi)| / (hi - lo)."""
    F, P = 1000, 1000
    rnd = po.draw_randoms_philox(2 ** 32 + 5, 1, 2, F, P, 2, [0, 1], 1, 9, 0.1)
    bbox = torch.tensor([[3.3, 17.8, 0.6, 9.1]] * 2)
    iw, ih = so.pixel_indices(rnd["kf"], rnd["u_w"], rnd["u_h"], bbox)
    for idx, lo, hi in ((iw, 3.3, 17.8), (ih, 0.6, 9.1)):
        ks = np.arange(int(np.floor(lo)), int(np.ceil(hi)))
        p = np.array([min(k + 1, hi) - max(k, lo) for k in ks]) / (hi - lo)
        counts = np.array([(idx == k).sum().item() for k in ks])
        assert counts.sum() == F * P
        assert stats.chisquare(counts, p * F * P).pvalue > P_MIN
    # independence of the two coordinates: a 2-D contingency table of column x row
    table = np.histogram2d(iw.flatten().numpy(), ih.flatten().numpy(), bins=(np.arange(3, 19), np.arange(0, 11)))[0]
    table = table[table.sum(1) > 0][:, table.sum(0) > 0]
    assert stats.chi2_contingency(table).pvalue > P_MIN


def test_normals_are_gaussian_and_clip_at_the_expected_rate():
    """Box-Muller normals: KS against N(0, eps/3) before clipping, and the fraction clipped at +-eps (the 3-sigma
    tails, 0.27 %) as a binomial count."""
    eps = 0.1
    nrm = po.draw_randoms_philox(123, 0, 0, 1000, 1000, 3, [1, 2], 1, 9, eps)["nrm"].numpy().ravel()
    assert nrm.size == 9 * 10 ** 6
    sd = float(np.float32(eps) / np.float32(3))
    assert stats.kstest(nrm, stats.norm(0.0, sd).cdf).pvalue > P_MIN
    clipped = int((np.abs(nrm) > np.float32(eps)).sum())
    assert stats.binomtest(clipped, nrm.size, 2 * stats.norm.sf(3.0)).pvalue > P_MIN
    # the four words of a chunk are four independent normals: neighbouring columns uncorrelated
    m = nrm.reshape(-1, 9)
    for j in range(8):
        assert abs(np.corrcoef(m[:, j], m[:, j + 1])[0, 1]) < 5 / np.sqrt(m.shape[0])


def test_streams_objects_and_offsets_are_uncorrelated():
    n = 10 ** 6
    lim = 5 / np.sqrt(n)

    def uw(b, off, seed=7):
        return po.draw_randoms_philox(seed, off, b, 1000, 1000, 2, [0, 1], 1, 9, 0.1)["u_w"].numpy().ravel()

    a = uw(0, 0)
    for other in (uw(1, 0), uw(0, 1), uw(0, 0, seed=7 + 2 ** 32)):
        assert abs(np.corrcoef(a, other)[0, 1]) < lim
    # the keyframe stream against the pixel stream at the same index (c0 = f = i)
    k0, k1 = po.seed_key(7)
    i = np.arange(n, dtype=np.uint64)
    kf_u = po.u01(po.philox4x32_10(i, po.STREAM_KF, 0, 0, k0, k1)[0])
    assert abs(np.corrcoef(kf_u, a)[0, 1]) < lim
    uz = po.draw_randoms_philox(7, 0, 0, 1000, 1000, 2, [0, 1], 1, 9, 0.1)["u_z"].numpy()
    assert abs(np.corrcoef(uz[:, 0], a)[0, 1]) < lim and abs(np.corrcoef(uz[:, 0], uz[:, 4])[0, 1]) < lim


# ---- power: what the range checks cannot see -------------------------------------------------------------------------
def _golden_objects(n_kf=None, latest=None):
    g = np.load(os.path.join(GOLDEN, "sampler_obj.npz"))
    t = [torch.from_numpy(g[k]) for k in ("rgbs_batch", "depth_batch", "t_wc_batch", "bbox")]
    n_kf = int(g["n_kf"]) if n_kf is None else n_kf
    latest = [int(x) for x in g["latest"]] if latest is None else latest
    return [(*t, n_kf, latest)] * 3, torch.from_numpy(g["rays_dir"])


MUTANTS = {
    "offset_plus_1": dict(offset_shift=1),
    "objects_b_and_b1_swapped": dict(b_index=[1, 0, 3]),
    "seed_halves_swapped": dict(seed_fn=lambda s: ((s & 0xFFFFFFFF) << 32) | (s >> 32)),
    "streams_2_and_3_swapped": dict(streams=(0, 1, 3, 2)),
    "latest_rule_at_2_keyframes": dict(latest_from=2),
}


def mutant_launch(objects, rays, F, P, cfg, seed, offset, mutant=None):
    """One Philox-mode launch of the restatement, under the named wrong scheme (``None``: the kernel's)."""
    m = dict(MUTANTS[mutant]) if mutant else {}
    seed = m.pop("seed_fn", lambda s: s)(seed)
    offset = offset + m.pop("offset_shift", 0)
    return po.sample_philox(objects, F, P, rays, cfg, seed, offset, **m)


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_wrong_draw_schemes_pass_the_range_checks(mutant):
    """tests/test_sampler_gpu.py's Philox-mode checks accept every one of these wrong schemes: only an exact
    comparison tells them from the kernel's."""
    from tests.test_sampler_gpu import philox_mode_checks
    F, P, n1, n2, eps, oeps = 100, 24, 1, 9, 0.1, 0.05
    # the latest rule only differs from the kernel's at n_kf = 2
    objects, rays = _golden_objects(*((2, [1, 0]) if mutant == "latest_rule_at_2_keyframes" else (None, None)))
    cfg = so.SamplerCfg(n_bins_cam2surface=n1, n_bins=n2, surface_eps=eps, stop_eps=oeps)
    a = mutant_launch(objects, rays, F, P, cfg, 123, 0, mutant)
    b = mutant_launch(objects, rays, F, P, cfg, 123, 0, mutant)
    c = mutant_launch(objects, rays, F, P, cfg, 123, 1, mutant)
    philox_mode_checks(a, b, c, n1, n2, eps, oeps)
    right = mutant_launch(objects, rays, F, P, cfg, 123, 0)
    philox_mode_checks(right, right, mutant_launch(objects, rays, F, P, cfg, 123, 1), n1, n2, eps, oeps)
    assert not torch.equal(a["z"], right["z"])                      # and yet the draws are different
