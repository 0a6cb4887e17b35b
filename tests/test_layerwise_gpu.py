"""GPU parity of the layer-wise tensor-core path (hidden 64/128/256: background model, iMAP model)."""
import pytest
import torch

from oracle import scene
from oracle import vmap_oracle as vo
from tests._util import make_ensemble, rel_l2, to_dev

pytestmark = pytest.mark.gpu

TOL_RENDER = 1e-3
TOL_GRAD = 7e-2      # wide layers: fp16 operands + L1 sign flips on few rays (cosine stays > 0.998)


def cos_sim(a, b):
    a = torch.as_tensor(a).double().flatten().cpu(); b = torch.as_tensor(b).double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-300))


@pytest.mark.parametrize("cfg", [
    dict(B=1, H=128, R=96, S=14, scale=5.0, n1=5),       # separate background model (room0_vMAP.json: hidden_feature_size_bg)
    dict(B=1, H=256, R=100, S=10, scale=5.0, n1=5),      # BASELINE configs[0]
    dict(B=1, H=256, R=70, S=32, scale=5.0, n1=5),       # BASELINE configs[4] shape
    dict(B=2, H=64, R=50, S=10, scale=2.0, n1=1),        # several wide objects (host loop over objects)
])
def test_oracle_parity_layerwise(cfg):
    B, H, R, S = cfg["B"], cfg["H"], cfg["R"], cfg["S"]
    params = vo.init_params(B, H, seed=7)
    batch = vo.synthetic_batch(B, R, S, seed=11, n_cam2surf=cfg["n1"])
    orc = vo.OracleEnsemble(params, cfg["scale"])
    loss_ref, g_ref = orc.grads(batch)
    d_ref, _, c_ref, o_ref = orc.render(batch)
    ens = make_ensemble(params, cfg["scale"], H, impl="layerwise")
    db = to_dev(batch)
    d, v, c, o = ens.render(db)
    errs = dict(depth=rel_l2(d, d_ref), colour=rel_l2(c, c_ref), opacity=rel_l2(o, o_ref))
    print("render rel-L2", errs)
    assert max(errs.values()) < TOL_RENDER, errs
    ens.forward_backward(db)
    assert abs(float(ens.loss_terms[:, 3].sum()) - float(loss_ref)) < 2e-3 * abs(float(loss_ref))
    got = ens.stacked(ens.grads)
    gerr = {k: (rel_l2(got[k], g_ref[k]), cos_sim(got[k], g_ref[k])) for k in vo.ALL_KEYS}
    print("grad (rel-L2, cos)", gerr)
    for k, (e, cs) in gerr.items():
        assert e < TOL_GRAD and cs > 0.998, (k, e, cs)


def test_layerwise_training_tracks_oracle_and_keeps_image_in_sync():
    """AdamW rewrites the fp16 image the GEMMs read; after training, the layer-wise render must agree with
    the fp32 kernel run on the SAME (trained) master weights, and quality must match the oracle's."""
    B, H, R, S, steps = 1, 128, 240, 14, 200       # (the CPU oracle at H=128 is what takes the time here)
    params = vo.init_params(B, H, seed=5)
    orc = vo.OracleEnsemble(params, 5.0)
    ens = make_ensemble(params, 5.0, H, impl="layerwise")
    for it in range(steps):
        b = scene.sphere_batch(B, R, S, seed=2000 + it, n_cam2surf=5)
        orc.step(b); ens.step(to_dev(b))
    ens.check_status()
    held = scene.sphere_batch(B, 1000, S, seed=77, n_cam2surf=5)
    dh = to_dev(held)
    d_l, _, c_l, _ = ens.render(dh, impl="layerwise")
    d_f, _, c_f, _ = ens.render(dh, impl="fp32")
    assert rel_l2(d_l, d_f) < 1e-3 and rel_l2(c_l, c_f) < 1e-3
    d_o, _, c_o, _ = orc.render(held)
    psnr_o, derr_o = scene.quality(d_o, c_o, held)
    psnr_g, derr_g = scene.quality(d_l.cpu(), c_l.cpu(), held)
    print(f"oracle PSNR {psnr_o:.2f} depth err {derr_o:.4f} | layerwise PSNR {psnr_g:.2f} depth err {derr_g:.4f}")
    assert abs(psnr_g - psnr_o) < 0.5 and psnr_o > 12.0        # short run on a noisy objective; see test_train_gpu.py for the 0.2 dB bar


def test_layerwise_speed_vs_fp32_kernel_imap_shape():
    B, H, R, S = 1, 256, 4800, 32          # BASELINE configs[4]: one rank's share would be 600 rays; full batch here
    params = vo.init_params(B, H, seed=1)
    db = to_dev(vo.synthetic_batch(B, R, S, seed=2, n_cam2surf=5))
    out = {}
    for impl in ("layerwise", "fp32"):
        ens = make_ensemble(params, 5.0, H, impl=impl)
        for _ in range(2):
            ens.step(db)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 5 if impl == "layerwise" else 2
        e0.record()
        for _ in range(n):
            ens.step(db)
        e1.record(); torch.cuda.synchronize()
        out[impl] = e0.elapsed_time(e1) / n
    flop = 6 * (4 * H * H + 220 * H + 63) * R * S
    print(f"iMAP step 1 x {R} x {S}, H={H}: layerwise {out['layerwise']:.2f} ms ({flop / out['layerwise'] / 1e9:.0f} TFLOP/s), "
          f"fp32 kernel {out['fp32']:.2f} ms")
    assert out["layerwise"] < out["fp32"]


@pytest.mark.parametrize("H,N", [(128, 3000), (64, 300001), (256, 1000)])
def test_eval_points_layerwise_forward_matches_oracle(H, N):
    """Trainer.eval_points (trainer.py:77-90) on the layer-wise wgmma GEMMs; N = 300001 crosses the internal
    262144-point chunking used to bound the activation workspace for 256^3 grids."""
    params = vo.init_params(1, H, seed=11)
    pts = (torch.rand(1, N, 3, generator=torch.Generator().manual_seed(2)) - 0.5) * 8
    alpha_ref, col_ref = vo.forward(params, torch.full((1,), 5.0), pts.view(1, N, 1, 3))
    ens = make_ensemble(params, 5.0, H, impl="layerwise")
    alpha, col = ens.eval_points(pts.cuda())
    a32, c32 = ens.eval_points(pts.cuda(), impl="fp32")
    assert rel_l2(a32, alpha_ref.view(1, N)) < 1e-4
    print(f"H={H} eval_points layer-wise vs oracle: alpha", rel_l2(alpha, alpha_ref.view(1, N)), "colour", rel_l2(col, col_ref.view(1, N, 3)))
    assert rel_l2(alpha, alpha_ref.view(1, N)) < 3e-3
    assert rel_l2(col, col_ref.view(1, N, 3)) < 1e-3
