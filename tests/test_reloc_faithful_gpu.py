"""Relocalisation scoring (vmb_reloc_score / vmb_reloc_select) against references computed outside the kernel, with
many hypotheses per CTA.

test_reloc_gpu.py compares each score with the tracker's iteration-1 loss at a handful of poses, where every CTA of
``k_reloc_fused`` holds one hypothesis. Here one call scores a table of several hundred, so each CTA keeps its weight
image, mask counts, samples and ``red`` across a chunk of them (``chunk >= 2`` is asserted on every call that must
exercise it), and about a dozen hypotheses per table -- the first, the last, the edges and the interior of chunks --
are checked per object and per term against the fp16-faithful restatement (oracle/track_fused_oracle.py, from the
kernel's own embedding), per hypothesis against the fp64 loss (oracle/track_oracle.py) and bit for bit against
``track_samples``. Also: sample counts that leave idle lanes, a stack wider than the reduction's 256 threads, several
groups on one or two handles, non-finite poses and empty masks inside a chunk, the workspace after a capture,
``relocalise`` against a restatement of its rounds, and ``select`` at its limits.

Run with -s to see every measured value next to its bar.
"""
import numpy as np
import pytest
import torch

from oracle import track_fused_oracle as tfo
from oracle import track_oracle as to
from oracle import vmap_oracle as vo
from tests.test_fused_faithful_gpu import probe_embedding
from tests.test_reloc_oracle import select_order
from tests.test_track_fused_gpu import SCALE, _rand_pose, _stack

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEEDS = (0, 1, 2)
N_TABLE = 384
# rays per shape: never a multiple of k_reloc_fused's tile (4 * (32 // S) rays) nor of K10's (128 // S)
R_OF_S = {5: 61, 7: 45, 10: 61, 14: 47, 17: 37, 32: 33}

# Bars, 4-5x the worst an H100 80GB HBM3 (700 W) measured over the shapes and seeds below (the tests print them):
#   per (hypothesis, object, term) error against the fp16-faithful restatement from the kernel's embedding, relative to
#   the term or TERM_FLOOR, whichever is larger: worst 6.0e-4 (S 10, B 20).  The floor is for terms near 0, such as
#   the opacity term of an object whose rays all saturate: the kernel's fp32 sigmoids resolve 1 - O to about 6e-8 a
#   ray, so such a term is 1e-8 on the GPU and 1e-10 in fp64 (measured: 1.7e-8 against 1.0e-10, K10 3.5e-8);
#   per hypothesis, the score's relative error against the fp64 loss: worst 2.7e-3 (S 32, B 1);
#   several groups, the score against the multi-group tracker's loss (one tree over every group's objects instead of
#   one per group, k_reloc.cuh), relative: worst 3.2e-16.
FAITHFUL_TERM_BAR, TERM_FLOOR = 2.5e-3, 1e-4
ORACLE_LOSS_BAR = 1.2e-2
MULTI_GROUP_BAR = 1.5e-15


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _chunk(n_hyp, B, R, S):
    """launch_reloc_fused's hypotheses per CTA: enough CTAs for about four waves of two per SM."""
    nr = 4 * (32 // S)
    ctas = -(-R // nr) * B
    want = max(1, min(n_hyp, -(-8 * _n_sm() // ctas)))
    return -(-n_hyp // want)


def _table(seed, n=N_TABLE):
    """[n, 4, 4] device fp64: the identity, _rand_pose draws, then ``hypotheses`` composed on a prior."""
    from vmap_b200.reloc import _compose, hypotheses
    n_rand = n // 3
    P = torch.from_numpy(np.stack([np.eye(4)] + [_rand_pose(1000 * seed + i) for i in range(1, n_rand)])).to(DEV)
    prior = torch.from_numpy(_rand_pose(1000 * seed + 999, 10.0, 0.1)).to(DEV)[None]
    D = torch.from_numpy(hypotheses(n - n_rand, 30.0, 0.3).copy()).to(DEV)
    return torch.cat([P, _compose(prior, D).reshape(-1, 4, 4)]).contiguous()


def _sampled(n, chunk, extra=()):
    """About a dozen hypotheses: the first, the last, and the first, an interior one and the last of some chunks."""
    mid = (n // chunk // 2) * chunk
    last = ((n - 1) // chunk) * chunk
    idx = {0, 1, chunk - 1, chunk, mid, mid + chunk // 2, mid + chunk - 1, n // 3, last, n - 2, n - 1, *extra}
    return sorted(i for i in idx if 0 <= i < n)


def _setup(B, R, S, seed, **kw):
    from vmap_b200.reloc import Relocalizer
    from vmap_b200.track import SampleGroup
    ens, rows, batch, og = _stack(B, R, S, seed=seed)
    sg = SampleGroup(ens, rows, batch, 1, impl="fused")
    kw = {"n_hyp": 16, "top_k": 4, **kw}
    return ens, rows, batch, og, sg, Relocalizer([sg], **kw)


def _tracker_losses(groups, P):
    """track_samples' iteration-1 loss from each pose of P [k, 4, 4]: one iteration at zero rates."""
    from vmap_b200.track import track_samples
    return np.array([float(track_samples(groups, P[h].cpu().numpy(), 1, 0.0, 0.0, record=False)["losses"][0])
                     for h in range(P.shape[0])])


def _faithful_terms(og, P):
    """[k, B, 4] per-object terms of the fp16-faithful restatement at each pose of P [k, 4, 4], from the kernel's own
    embedding at pose_point's points: the k x B objects go in one call, object h * B + b posed by P[h]."""
    T = P.cpu().numpy()
    k = T.shape[0]
    b = og["batch"]
    B, R, S, _ = b["pcs"].shape
    rep = lambda v: v.repeat(k, *([1] * (v.dim() - 1)))                    # noqa: E731
    params = {n: rep(v) for n, v in og["params"].items()}
    batch = {n: rep(v) for n, v in b.items()}
    frames = torch.arange(k).repeat_interleave(B)[:, None].expand(k * B, R).contiguous()
    t, _ = tfo.posed_points(T, frames, batch["pcs"].double(), SCALE)
    pts = (t * SCALE).float().reshape(k * B, R * S, 3).to(DEV).contiguous()   # exact: SCALE is a power of two
    e1, e2 = probe_embedding(params, SCALE, pts)
    f = tfo.evaluate(params, torch.full((k * B,), SCALE), batch, T, frames, emb=(e1.cpu(), e2.cpu()))
    return f["terms"].reshape(k, B, 4).numpy()


def _oracle_losses(og, P):
    """The fp64 loss at each pose of P (track_oracle.evaluate's loss, without its gradient)."""
    return np.array([to.loss_at([og], P[h].cpu().numpy()) for h in range(P.shape[0])])


def _rel_each(a, b):
    return np.abs(a - b) / np.abs(b)


def _term_err(a, b):
    return np.abs(a - b) / np.maximum(np.abs(b), TERM_FLOOR)


# ---- 1 + 2. per hypothesis, per object, per term against the references, and bit for bit against the tracker -------

SHAPES = [(S, B) for S in (5, 7, 10, 14, 17, 32) for B in (1, 3, 20)]


@pytest.mark.parametrize("S,B", SHAPES, ids=[f"S{S}B{B}" for S, B in SHAPES])
def test_scores_against_the_references_and_the_tracker(S, B):
    R = R_OF_S[S]
    worst = [0.0, 0.0]
    for seed in SEEDS:
        ens, rows, batch, og, sg, rl = _setup(B, R, S, seed=13 * S + B + 100 * seed)
        P = _table(seed)
        chunk = _chunk(N_TABLE, B, R, S)
        assert chunk >= 2, chunk
        terms = torch.full((N_TABLE, B, 4), float("nan"), dtype=torch.float64, device=DEV)
        scores = rl.score(P, terms).cpu().numpy()
        t = terms.cpu().numpy()
        assert np.all(np.isfinite(scores)) and np.all(np.isfinite(t))
        idx = _sampled(N_TABLE, chunk, extra=(N_TABLE // 3 + 1,))
        # bit for bit: the tracker's iteration-1 loss from the same pose, whatever the hypothesis's place in its chunk
        trk = _tracker_losses([sg], P[idx])
        assert np.array_equal(scores[idx], trk), (idx, scores[idx] - trk)
        # per object, per term: the fp16-faithful restatement; per hypothesis: the fp64 loss
        f = _faithful_terms(og, P[idx])
        worst[0] = max(worst[0], _term_err(t[idx], f).max())
        worst[1] = max(worst[1], _rel_each(scores[idx], _oracle_losses(og, P[idx])).max())
    print(f"S{S} B{B} R{R} chunk {chunk}: vs faithful terms {worst[0]:.2e} (bar {FAITHFUL_TERM_BAR:.1e}); "
          f"vs fp64 loss {worst[1]:.2e} (bar {ORACLE_LOSS_BAR:.1e})")
    assert worst[0] <= FAITHFUL_TERM_BAR and worst[1] <= ORACLE_LOSS_BAR, worst


@pytest.mark.parametrize("S", sorted(R_OF_S))
def test_score_does_not_depend_on_the_batch(S):
    """The same poses score the same alone, in a table of several hundred and at two offsets in a table of 4096: their
    place in a CTA's chunk and the chunk size do not change a bit."""
    from vmap_b200 import _lib
    R, B = R_OF_S[S], 3
    ens, rows, batch, og, sg, rl = _setup(B, R, S, seed=7 + S)
    P = _table(S)
    mid = rl.score(P).cpu().numpy()
    assert _chunk(N_TABLE, B, R, S) >= 2 and _chunk(4096, B, R, S) >= 2
    filler = torch.from_numpy(np.stack([_rand_pose(50_000 + i) for i in range(4096 - N_TABLE)])).to(DEV)
    for off in (4096 - N_TABLE, 4096 - N_TABLE - 5):
        big = rl.score(torch.cat([filler[:off], P, filler[off:]])).cpu().numpy()
        assert np.array_equal(big[off:off + N_TABLE], mid), off
    for h in _sampled(N_TABLE, _chunk(N_TABLE, B, R, S)):
        assert np.array_equal(rl.score(P[h:h + 1]).cpu().numpy(), mid[h:h + 1]), h
    assert int(rl.status[0]) & ~_lib.TRACK_ST_CLAMP == 0


# ---- 3. a stack wider than k_reloc_reduce's 256 threads ---------------------------------------------------------------

def test_wide_stack():
    S, B, R, H = 10, 300, 13, 24
    ens, rows, batch, og, sg, rl = _setup(B, R, S, seed=31)
    P = _table(3)[::16][:H].contiguous()
    chunk = _chunk(H, B, R, S)
    assert chunk >= 2, chunk
    terms = torch.zeros(H, B, 4, dtype=torch.float64, device=DEV)
    scores = rl.score(P, terms).cpu().numpy()
    t = terms.cpu().numpy()
    idx = _sampled(H, chunk)
    assert np.all(np.isfinite(scores)) and np.array_equal(scores[idx], _tracker_losses([sg], P[idx]))
    some = [0, chunk // 2, H - 1]
    err = _term_err(t[some], _faithful_terms(og, P[some])).max()
    print(f"S{S} B{B} R{R} chunk {chunk}: vs faithful terms {err:.2e} (bar {FAITHFUL_TERM_BAR:.1e})")
    assert err <= FAITHFUL_TERM_BAR


# ---- 4. several groups ---------------------------------------------------------------------------------------------

def _three_groups(seed):
    """Two groups of different B x R (and S) on one handle, the smaller first, and a third on a second handle."""
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.track import SampleGroup
    ens = []
    for n in (10, 6):
        e = VmapEnsemble(n, hidden=32, scale=SCALE, impl="fp32")
        e.load_stacked(vo.init_params(n, 32, seed=seed + n))
        ens.append(e)
    spec = ((ens[0], [1, 2, 3], 40, 10), (ens[0], [4, 5, 6, 7, 8], 61, 14), (ens[1], [0, 1, 2, 3], 33, 32))
    groups = []
    for i, (e, rows, R, S) in enumerate(spec):
        b = vo.synthetic_batch(len(rows), R, S, seed=seed + 10 * i, n_cam2surf=S - 9 if S > 9 else 1)
        groups.append((SampleGroup(e, rows, b, 1, impl="fused"), len(rows), R, S))
    return groups


def test_several_groups():
    from vmap_b200 import _lib
    from vmap_b200.reloc import Relocalizer
    gs = _three_groups(seed=4)
    groups = [g for g, _, _, _ in gs]
    P = _table(5, n=256)
    for _, B, R, S in gs:
        assert _chunk(256, B, R, S) >= 2
    rl = Relocalizer(groups, n_hyp=16, top_k=4)
    s = rl.score(P)
    parts = [Relocalizer([g], n_hyp=16, top_k=4).score(P).cpu().numpy() for g in groups]
    total = np.zeros(256)
    for p in parts:
        total = total + p                                  # scores[h] += ..., group by group in call order
    sn = s.cpu().numpy()
    assert np.all(np.isfinite(sn)) and np.array_equal(sn, total)
    idx = _sampled(256, _chunk(256, gs[0][1], gs[0][2], gs[0][3]))
    trk = _tracker_losses(groups, P[idx])
    err = np.abs(sn[idx] - trk).max() / np.abs(trk).min()
    print(f"three groups: vs the multi-group tracker's loss, relative {err:.2e} (bar {MULTI_GROUP_BAR:.0e})")
    assert err <= MULTI_GROUP_BAR
    # eager, then a capture and its replay
    out = {}
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        rl.score(P)
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out["s"] = rl.score(P)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out["s"], s)
    assert int(rl.status[0]) & ~_lib.TRACK_ST_CLAMP == 0
    # per-object terms belong to one group: with several, the second call would overwrite the first's rows
    terms = torch.zeros(256, gs[0][1], 4, dtype=torch.float64, device=DEV)
    with pytest.raises(_lib.VmbError):
        rl.score(P, terms)
    assert torch.all(terms == 0)


# ---- 5. non-finite poses, empty masks and a bad row inside a chunk ----------------------------------------------------

def test_non_finite_poses_inside_a_chunk():
    """Non-finite poses reach only arithmetic (pose_point, the PE's range reduction and MUFU sin / cos, the network, the
    render and the loss): no index or bound comes from a coordinate.  Their scores are non-finite, and the hypotheses
    after them in the same CTA score exactly as without them."""
    from vmap_b200 import _lib
    S, B = 10, 3
    R = R_OF_S[S]
    ens, rows, batch, og, sg, rl = _setup(B, R, S, seed=61)
    P = _table(6)
    chunk = _chunk(N_TABLE, B, R, S)
    assert chunk >= 4, chunk
    c0 = 10 * chunk
    bad = P.clone()
    bad[c0 + 1, 0, 3] = float("nan")
    bad[c0 + 2, 1, 1] = float("inf")
    clean = rl.score(P).cpu().numpy()
    s = rl.score(bad).cpu().numpy()
    keep = np.ones(N_TABLE, bool)
    keep[[c0 + 1, c0 + 2]] = False
    assert not np.isfinite(s[c0 + 1]) and not np.isfinite(s[c0 + 2])
    assert np.array_equal(s[keep], clean[keep])
    sl = slice(c0, c0 + chunk)
    idx, out = rl.select(torch.from_numpy(s[sl]).to(DEV), bad[sl], chunk)
    assert idx.cpu().tolist() == select_order(s[sl], chunk) and idx.cpu().tolist()[-2:] == [1, 2]
    assert torch.equal(out[:-2], bad[sl][idx[:-2].long()])
    assert int(rl.status[0]) & ~_lib.TRACK_ST_CLAMP == 0


def test_empty_masks_and_a_bad_row_inside_a_chunk():
    from vmap_b200 import _lib
    from vmap_b200.reloc import Relocalizer
    from vmap_b200.track import SampleGroup
    S, B = 14, 5
    R = R_OF_S[S]
    ens, rows, batch, og, sg, rl = _setup(B, R, S, seed=71)
    P = _table(7)
    chunk = _chunk(N_TABLE, B, R, S)
    assert chunk >= 2, chunk
    t0 = torch.zeros(N_TABLE, B, 4, dtype=torch.float64, device=DEV)
    s0 = rl.score(P, t0).cpu().numpy()
    t0 = t0.cpu().numpy()
    # object 0: no valid depth ray; object 1: no sem != 0 ray; object 2: no sem != 2 ray; objects 3, 4 unchanged
    b2 = {k: v.clone() for k, v in batch.items()}
    b2["mask_depth"][0] = False
    b2["sem"][1] = 0
    b2["sem"][2] = 2
    sg2 = SampleGroup(ens, rows, b2, 1, impl="fused")
    rl2 = Relocalizer([sg2], n_hyp=16, top_k=4)
    t2 = torch.zeros(N_TABLE, B, 4, dtype=torch.float64, device=DEV)
    s2 = rl2.score(P, t2).cpu().numpy()
    t2 = t2.cpu().numpy()
    assert np.all(t0[:, :3, :3] != 0.0)
    assert np.all(t2[:, 0, 0] == 0.0) and np.all(t2[:, 1, :2] == 0.0) and np.all(t2[:, 2, 2] == 0.0)
    assert np.array_equal(t2[:, 0, 1:3], t0[:, 0, 1:3])
    assert np.array_equal(t2[:, 3:], t0[:, 3:])
    idx = _sampled(N_TABLE, chunk)
    assert np.array_equal(s2[idx], _tracker_losses([sg2], P[idx]))
    og2 = dict(og, batch=b2)
    err = _term_err(t2[idx], _faithful_terms(og2, P[idx])).max()
    print(f"empty masks, S{S} B{B} chunk {chunk}: vs faithful terms {err:.2e} (bar {FAITHFUL_TERM_BAR:.1e})")
    assert err <= FAITHFUL_TERM_BAR
    # a row outside the stack: that object contributes nothing at every hypothesis, the others are unchanged
    sg.rows_dev[1] = ens.n_obj + 5
    tb = torch.zeros(N_TABLE, B, 4, dtype=torch.float64, device=DEV)
    bad = rl.score(P, tb).cpu().numpy()
    tb = tb.cpu().numpy()
    assert int(rl.status[0]) & _lib.TRACK_ST_BAD_ROW
    assert np.all(tb[:, 1] == 0.0) and np.array_equal(tb[:, [0, 2, 3, 4]], t0[:, [0, 2, 3, 4]])
    assert np.all(bad < s0)


# ---- 6. the workspace after a capture ---------------------------------------------------------------------------------

def test_workspace_after_a_capture():
    from vmap_b200 import _lib
    S, B = 10, 3
    ens, rows, batch, og, sg, rl = _setup(B, 40, S, seed=81)
    P = _table(8)
    eager = rl.score(P[:200])
    out = {}
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        rl.score(P[:200])
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out["s"] = rl.score(P[:200])
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out["s"], eager)
    # the graph holds the workspace: a call needing more rays is refused (eagerly), not given a moved buffer
    with pytest.raises(_lib.VmbError, match="operation not permitted when stream is capturing"):
        rl.score(P)
    out["s"].zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out["s"], eager)
    assert torch.equal(rl.score(P[:50]), eager[:50])


# ---- 7. relocalise against a restatement of its rounds ---------------------------------------------------------------

def test_relocalise_against_a_restatement_of_its_rounds():
    from vmap_b200.reloc import _compose
    S, B = 10, 3
    R = R_OF_S[S]
    ens, rows, batch, og, sg, rl = _setup(B, R, S, seed=91, n_hyp=200, top_k=8, rot_deg=30.0, trans=0.3)
    priors = torch.from_numpy(np.stack([_rand_pose(92), _rand_pose(93)])).to(DEV)
    extra = torch.from_numpy(np.stack([_rand_pose(94), np.eye(4), _rand_pose(95)])).to(DEV)
    K = rl.top_k
    assert _chunk(2 * rl.n_hyp, B, R, S) >= 2 and _chunk(K * rl.n_hyp, B, R, S) >= 2
    calls = []                                             # what relocalise scored and selected, in order
    score, select = rl.score, rl.select
    rl.score = lambda p, *a: calls.append(("score", p.clone(), score(p, *a))) or calls[-1][2]
    rl.select = lambda s, p, k: calls.append(("select", select(s, p, k))) or calls[-1][1]
    pose, best, top = rl.relocalise(priors, extra)
    del rl.score, rl.select
    torch.cuda.synchronize()
    # the restatement: round 1 around the priors, round 2 around its top K, then the pick with the extra candidates
    h1 = _compose(priors, rl.D1).reshape(-1, 4, 4)
    s1 = rl.score(h1).cpu().numpy()
    o1 = select_order(s1, K)
    h2 = _compose(h1[o1], rl.D2).reshape(-1, 4, 4)
    s2 = rl.score(h2).cpu().numpy()
    o2 = select_order(s2, K)
    se = rl.score(extra).cpu().numpy()
    cand = torch.cat([h1[o1], h2[o2], extra])
    sc = np.concatenate([s1[o1], s2[o2], se])
    o = select_order(sc, K)
    kinds = [c[0] for c in calls]
    assert kinds == ["score", "select", "score", "select", "score", "select"], kinds
    assert torch.equal(calls[0][1], h1) and np.array_equal(calls[0][2].cpu().numpy(), s1)
    assert calls[1][1][0].cpu().tolist() == o1 and torch.equal(calls[1][1][1], h1[o1])
    assert torch.equal(calls[2][1], h2) and np.array_equal(calls[2][2].cpu().numpy(), s2)
    assert calls[3][1][0].cpu().tolist() == o2 and torch.equal(calls[3][1][1], h2[o2])
    assert calls[5][1][0].cpu().tolist() == o
    assert torch.equal(pose, cand[o[0]]) and float(best) == sc[o[0]] and np.array_equal(top.cpu().numpy(), sc[o])
    print(f"relocalise: round 1 best {s1[o1[0]]:.5f}, round 2 best {s2[o2[0]]:.5f}, extra best {se.min():.5f} "
          f"-> {float(best):.5f}")


# ---- 8. select at its limits, and the guards ----------------------------------------------------------------------

def test_select_at_its_limits():
    ens, rows, batch, og, sg, rl = _setup(1, 20, 10, seed=2)
    rng = np.random.default_rng(3)
    for n in (1, 255, 256, 257, 4095, 4096):
        P = torch.from_numpy(rng.normal(size=(n, 4, 4))).to(DEV)
        cases = {"ties": np.round(rng.normal(size=n), 1), "nan": np.full(n, np.nan),
                 "inf": rng.choice([np.inf, -np.inf, 1.0, -1.0, np.nan], size=n),
                 "zeros": rng.choice([0.0, -0.0, 1.0, -1.0], size=n, p=[0.4, 0.4, 0.1, 0.1])}
        for name, s in cases.items():
            for k in sorted({1, min(n, 7), min(n, 64)}):
                idx, poses = rl.select(torch.from_numpy(s).to(DEV), P, k)
                want = select_order(s, k)
                assert idx.cpu().tolist() == want, (n, name, k)
                assert torch.equal(poses, P[want]), (n, name, k)


class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called: a guard let bad arguments through")


def test_guards_raise_before_any_launch():
    from vmap_b200 import _lib
    ens, rows, batch, og, sg, rl = _setup(3, 20, 10, seed=3)
    P = _table(9, n=6)
    s = rl.score(P)
    f64 = dict(dtype=torch.float64, device=DEV)
    lib, ens.lib = ens.lib, _NoLaunch()
    try:
        bad_score = [
            (P.cpu(), None), (P[:, :, :3], None), (P.reshape(6, 16), None), (P.reshape(2, 3, 4, 4), None),
            (P.long(), None), (P, torch.zeros(6, 3, 4, dtype=torch.float64)), (P, torch.zeros(6, 3, 4, **f64).float()),
            (P, torch.zeros(6, 2, 4, **f64)), (P, torch.zeros(5, 3, 4, **f64)), (P, torch.zeros(6, 3, 5, **f64)),
            (P, torch.zeros(4, 3, 6, **f64).permute(2, 1, 0)), (P, torch.zeros(6 * 3 * 4, **f64))]
        for poses, terms in bad_score:
            with pytest.raises(_lib.VmbError):
                rl.score(poses, terms)
        bad_select = [
            (s.cpu(), P, 2), (s.float(), P, 2), (s[None], P, 2), (s[:0], P[:0], 1), (s, P[:5], 2), (s, P.float(), 2),
            (s, P.cpu(), 2), (s, P.reshape(6, 16), 2), (s, P, 0), (s, P, 7), (s, P, 2.5),
            (torch.zeros(_lib.RELOC_MAX_HYP + 1, **f64), torch.zeros(_lib.RELOC_MAX_HYP + 1, 4, 4, **f64), 2)]
        for scores, poses, k in bad_select:
            with pytest.raises(_lib.VmbError):
                rl.select(scores, poses, k)
    finally:
        ens.lib = lib
    idx, _ = rl.select(s, P, 6)
    assert idx.cpu().tolist() == select_order(s.cpu().numpy(), 6)
