"""Parity at the shapes BASELINE.json names (configs[0..4]); configs[1] is the bench workload and is
covered in test_umma_gpu.py.  The reference is the CPU oracle at the full shape (a few seconds per case)."""
import pytest
import torch

from oracle import vmap_oracle as vo
from tests._util import make_ensemble, rel_l2, to_dev

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("impl", ["fp32", "auto"])
def test_cfg0_imap_single_mlp_h256_100rays(impl):
    """configs[0]: iMAP single-scene MLP, 1 object, 100 rays x 10 samples, hidden 256 (CPU-runnable).
    "fp32" is the CUDA-core parity anchor; "auto" resolves to the layer-wise tensor-core path (fp16 operands)."""
    params = vo.init_params(1, 256, seed=0)
    batch = vo.synthetic_batch(1, 100, 10, seed=1, n_cam2surf=5)
    orc = vo.OracleEnsemble(params, 5.0)
    ens = make_ensemble(params, 5.0, 256, impl=impl)
    db = to_dev(batch)
    tol_loss, tol_par = (2e-4, 1e-4) if impl == "fp32" else (3e-3, 2e-2)
    for _ in range(3):
        l_ref = float(orc.step(batch))
        l = float(ens.step(db))
        assert abs(l - l_ref) < tol_loss * abs(l_ref)
    for k in vo.ALL_KEYS:      # Adam normalises near-zero gradients, so atomics-order noise shows up at ~1e-5
        assert rel_l2(ens.view(k), orc.params[k]) < tol_par, k


@pytest.mark.parametrize("n_obj", [50, 160])
def test_cfg2_cfg3_many_objects_umma_vs_oracle(n_obj):
    """configs[2] (50 objects x 1200 rays) and configs[3] (160 objects = 8 x 20): every CTA walks several objects.
    Reference = the CPU oracle at the full shape."""
    R, S = 1200 if n_obj == 50 else 240, 10
    params = vo.init_params(n_obj, 32, seed=2)
    batch = vo.synthetic_batch(n_obj, R, S, seed=3)
    db = to_dev(batch)
    orc = vo.OracleEnsemble(params, 2.0)
    d_a, _, c_a, o_a = orc.render(batch)
    _, g_ref = orc.grads(batch)
    lt_ref = orc.loss_terms(batch).cuda()                      # [B,4] per-object terms
    u = make_ensemble(params, 2.0, 32, impl="umma")
    d_u, _, c_u, o_u = u.render(db)
    assert rel_l2(d_u, d_a) < 1e-3 and rel_l2(c_u, c_a) < 1e-3 and rel_l2(o_u, o_a) < 1e-3
    u.forward_backward(db)
    # per-object losses agree object by object (no cross-object leakage when CTAs straddle objects)
    lt = float(((lt_ref - u.loss_terms).abs() / (lt_ref.abs() + 1e-6)).max())
    print('max per-object loss-term rel diff', lt)
    assert lt < 3e-2
    for k in vo.ALL_KEYS:
        ga, gu = g_ref[k].cuda(), u.view(k, u.grads)
        per_obj = ((ga - gu).flatten(1).norm(dim=1) / (ga.flatten(1).norm(dim=1) + 1e-20))
        # The losses are L1: d|x|/dx = sign(x) flips for rays whose residual is within the fp16 forward noise,
        # so a few objects with few contributing rays show large relative differences (deterministic);
        # the bulk must agree closely and the whole-stack gradient within the kernel's bar.
        q90 = float(per_obj.kthvalue(max(1, int(0.9 * n_obj))).values)
        print(k, 'per-object grad rel-L2: median', float(per_obj.median()), 'p90', q90, 'max', float(per_obj.max()),
              'stack', rel_l2(gu, ga))
        assert float(per_obj.median()) < 3e-2 and q90 < 0.1 and float(per_obj.max()) < 0.6, (k, float(per_obj.max()))
        assert rel_l2(gu, ga) < 6e-2, k
    # independence: permuting the objects permutes the results
    perm = torch.randperm(n_obj, generator=torch.Generator().manual_seed(0))
    pp = {k: v[perm] for k, v in params.items()}
    dbp = {k: v[perm.to(v.device)].contiguous() for k, v in db.items()}
    u2 = make_ensemble(pp, 2.0, 32, impl="umma")
    u2.forward_backward(dbp)
    assert rel_l2(u2.loss_terms, u.loss_terms[perm.cuda()]) < 1e-5


def test_cfg4_imap_h256_32_samples():
    """configs[4] shape: whole-scene MLP, hidden 256, 32 samples per ray (rays reduced for the oracle)."""
    params = vo.init_params(1, 256, seed=4)
    batch = vo.synthetic_batch(1, 96, 32, seed=5, n_cam2surf=5)
    orc = vo.OracleEnsemble(params, 5.0)
    loss_ref, g_ref = orc.grads(batch)
    ens = make_ensemble(params, 5.0, 256)
    db = to_dev(batch)
    d, _, c, _ = ens.render(db)
    d_ref, _, c_ref, _ = orc.render(batch)
    assert rel_l2(d, d_ref) < 2e-5 and rel_l2(c, c_ref) < 2e-5
    ens.forward_backward(db)
    assert abs(float(ens.loss_terms[:, 3].sum()) - float(loss_ref)) < 5e-5 * abs(float(loss_ref))
    for k in vo.ALL_KEYS:
        assert rel_l2(ens.view(k, ens.grads), g_ref[k]) < 3e-4, k
