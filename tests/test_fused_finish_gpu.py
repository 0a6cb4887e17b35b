"""The finish of the fused hidden-32 step (k_step_fused): each object's partial rows are reduced and AdamW applied as soon
as that object's last segment lands, by whichever CTA claims the chunk.  On shapes whose segments land in very different
orders -- one object, several objects per CTA, the largest stack whose mask counts fit in shared memory, an object of
more than ten segments, every instantiation (S = 10, 14 and the generic one), the JOINT step, and object counts that
shrink and grow on one handle (the sync words must re-arm) -- the fused step must give the same bits as the unfused
path (the same kernel with fuse_adam off, then vmb_adam), and two fresh runs must give the same bits."""
import math

import numpy as np
import pytest
import torch

from oracle import vmap_oracle as vo
from tests._util import make_ensemble, to_dev

pytestmark = pytest.mark.gpu

# the largest stack whose mask counts fit in the kernel's shared memory: uf::MAX_OBJ_SMEM = (227 KB - uf::SM_CNT - 16) / 12,
# SM_CNT = activations 96256 + embedding gradient 36 * 2048 + weight image 26624 + heads 2048 + misc 512
MAX_OBJ_SMEM = (232448 - (96256 + 36 * 2048 + 26624 + 2048 + 512) - 16) // 12

SHAPES = [
    dict(B=1, R=300, S=10),                 # one object over 13+ CTAs: more than ten segments
    dict(B=300, R=12, S=10),                # one tile per object: two or three objects per CTA
    dict(B=MAX_OBJ_SMEM, R=12, S=10),       # the largest stack: about 21 objects per CTA
    dict(B=4, R=200, S=14),                 # SC = 14 instantiation
    dict(B=3, R=150, S=7),                  # SC = 0 instantiation
    dict(B=20, R=1200, S=10),               # BASELINE cfg 2
]
IDS = ["B{B}R{R}S{S}".format(**c) for c in SHAPES]
STATE = ("params", "exp_avg", "exp_avg_sq", "image", "step_counter", "loss_terms")


def batches_for(B, R, S, n, seed):
    return [to_dev(vo.synthetic_batch(B, R, S, seed=seed + i, n_cam2surf=1)) for i in range(n)]


def state(ens, n=None):
    n = ens.n_obj if n is None else n
    return {k: getattr(ens, k)[:n].clone() for k in STATE}


def assert_same(a, b, what):
    for k in STATE:
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs"


def fused_run(params, batches, steps):
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    for it in range(steps):
        ens.step(batches[it % len(batches)])
    torch.cuda.synchronize()
    ens.check_status()
    return state(ens)


def unfused_run(params, batches, steps):
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    for it in range(steps):
        ens.forward_backward(batches[it % len(batches)])
        ens.adam_step()
    torch.cuda.synchronize()
    ens.check_status()
    return state(ens)


@pytest.mark.parametrize("cfg", SHAPES, ids=IDS)
def test_fused_step_matches_unfused(cfg):
    """Three fused steps against forward_backward(fuse_adam=False) + adam_step, bit for bit, and a second fresh run of
    the fused step against the first."""
    B, R, S = cfg["B"], cfg["R"], cfg["S"]
    params = vo.init_params(B, 32, seed=7)
    batches = batches_for(B, R, S, 2, seed=70)
    f1 = fused_run(params, batches, 3)
    assert_same(f1, unfused_run(params, batches, 3), "fused vs unfused")
    assert_same(f1, fused_run(params, batches, 3), "two fresh fused runs")
    assert torch.equal(f1["step_counter"], torch.full((B,), 3, dtype=torch.int32, device="cuda"))


@pytest.mark.parametrize("cfg", [SHAPES[0], SHAPES[1], SHAPES[3]], ids=[IDS[0], IDS[1], IDS[3]])
def test_unfused_finish_accumulates(cfg):
    """fuse_adam off: the finish adds the reduced gradient into `grads`, so two calls give exactly the fp32 sum of the
    two calls' gradients taken alone, and the loss terms are those of the last call."""
    B, R, S = cfg["B"], cfg["R"], cfg["S"]
    params = vo.init_params(B, 32, seed=8)
    b1, b2 = batches_for(B, R, S, 2, seed=80)
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    ens.forward_backward(b1)
    g1 = ens.grads.clone()
    ens.grads.zero_()
    ens.forward_backward(b2)
    g2, l2 = ens.grads.clone(), ens.loss_terms.clone()
    ens.grads.copy_(g1)
    ens.forward_backward(b2)
    assert torch.equal(ens.grads, g1 + g2)
    assert torch.equal(ens.loss_terms, l2)


def test_object_count_changes_on_one_handle():
    """One handle runs launches of 6, 2, 6, 1 and 4 objects (rows 0..B-1 of its blocks), fused and, on a twin handle,
    unfused: every step agrees bit for bit, so the readiness counters, ticket and skip flags re-arm between launches
    whatever the object count."""
    Bmax, R, S = 6, 150, 10
    params = vo.init_params(Bmax, 32, seed=9)
    full = batches_for(Bmax, R, S, 1, seed=90)[0]
    fused = make_ensemble(params, 2.0, 32, impl="umma")
    twin = make_ensemble(params, 2.0, 32, impl="umma")
    for it, n in enumerate((6, 2, 6, 1, 4)):
        batch = {k: v[:n] for k, v in full.items()}
        for e in (fused, twin):
            e.n_obj = n
        fused.step(batch)
        twin.forward_backward(batch)
        twin.adam_step()
        torch.cuda.synchronize()
        assert_same(state(fused, n), state(twin, n), f"step {it} ({n} objects)")
    for e in (fused, twin):
        e.n_obj = Bmax
    want = torch.tensor([5, 4, 3, 3, 2, 2], dtype=torch.int32, device="cuda")
    assert torch.equal(fused.step_counter, want)


# ---- the JOINT instantiation -----------------------------------------------------------------------------------------

NPD = 10                                        # rays per draw


def _rand_pose(seed):
    from oracle import track_oracle as to
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    w *= math.radians(5.0) / np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w)
    T[:3, 3] = rng.uniform(-0.05, 0.05, 3)
    return T


def _joint_state(fuse_adam, B, R, S, seed):
    """Two joint steps (vmb_joint_step_fused) on a fresh B-object stack: AdamW inside the step, or fuse_adam off and
    adam_step after it."""
    from vmap_b200.ba import BaSampleGroup, ba_args
    from vmap_b200.ensemble import VmapEnsemble
    params = vo.init_params(B, 32, seed=seed)
    ens = VmapEnsemble(B, hidden=32, scale=2.0, impl="umma")
    ens.load_stacked(params)
    batch = vo.synthetic_batch(B, R, S, seed=seed + 1, n_cam2surf=1, empty_prob=(0.0, 0.0, 0.0, 0.0))
    n_draw = R // NPD
    kf_draw = np.stack([(np.arange(n_draw) + b) % 2 for b in range(B)]).astype(np.int32)
    kf_frame = np.array([[[1, 2], [0, 2], [1, 0]][b % 3] for b in range(B)], np.int32)
    P = np.stack([np.eye(4), _rand_pose(seed + 2), _rand_pose(seed + 3)])
    g = BaSampleGroup(ens, list(range(B)), batch, 1, NPD, kf_draw, kf_frame)
    f64 = dict(dtype=torch.float64, device="cuda")
    poses = torch.as_tensor(P, dtype=torch.float64).cuda().contiguous()
    win = torch.tensor([1, 2], dtype=torch.int32, device="cuda")
    adam = torch.zeros(2, 12, **f64)
    scratch = torch.zeros(8 * len(g.rows) * g.win + 12, **f64)
    status = torch.zeros(4, dtype=torch.int32, device="cuda")
    a = ba_args([g], 1, poses, win, 2, 0, adam, scratch, 0.0, 0.0, None, status)
    a.iter = 1
    g.bind(a.group[0], 0)
    batch = {k: v[:, :g.n_pix] for k, v in g.out.items()}
    for _ in range(2):
        ens.joint_step_fused(batch, a, 0, fuse_adam=fuse_adam)
        if not fuse_adam:
            ens.adam_step()
    torch.cuda.synchronize()
    ens.check_status()
    return state(ens)


@pytest.mark.parametrize("S", [10, 14])
def test_joint_fused_matches_unfused(S):
    B, R = 5, 70
    f1 = _joint_state(True, B, R, S, seed=21)
    assert_same(f1, _joint_state(False, B, R, S, seed=21), "joint fused vs unfused")
    assert_same(f1, _joint_state(True, B, R, S, seed=21), "two fresh joint runs")
