"""Trained-quality parity on a consistent scene (BASELINE target: trained PSNR within +-0.2 dB of the
reference on identical inputs): the CPU oracle (= the reference's fp32 functorch step) and the tensor-core
path train on the same batch stream from the same init; quality is measured on held-out rays."""
import pytest
import torch

from oracle import scene
from oracle import vmap_oracle as vo
from tests._util import make_ensemble, to_dev

pytestmark = pytest.mark.gpu


# fp32 CUDA-core kernel (any hidden size, parity anchor): same arithmetic as the oracle up to the order of its per-tile
# gradient atomics; over 600 L1-loss steps that noise occasionally moves the held-out PSNR by more than 0.05 dB (seen
# once in ~7 runs), so it shares the BASELINE bar of 0.2 dB.  The hidden-32 tensor-core path has no floating-point
# atomics and is bitwise reproducible (tests/test_umma_gpu.py::test_step_is_bitwise_reproducible).
@pytest.mark.parametrize("impl,tol_db", [("umma", 0.2), ("fp32", 0.2)])
def test_trained_psnr_matches_oracle(impl, tol_db):
    B, R, S, steps = 2, 240, 10, 600
    params = vo.init_params(B, 32, seed=5)
    orc = vo.OracleEnsemble(params, 2.0)
    ens = make_ensemble(params, 2.0, 32, impl=impl)
    for it in range(steps):
        b = scene.sphere_batch(B, R, S, seed=1000 + it)
        orc.step(b)
        ens.step(to_dev(b))
    ens.check_status()
    held = scene.sphere_batch(B, 2000, S, seed=99)
    d_o, _, c_o, _ = orc.render(held)
    d_g, _, c_g, _ = ens.render(to_dev(held))
    psnr_o, derr_o = scene.quality(d_o, c_o, held)
    psnr_g, derr_g = scene.quality(d_g.cpu(), c_g.cpu(), held)
    print(f"[{impl}] oracle PSNR {psnr_o:.2f} dB depth err {derr_o:.4f} | kernel PSNR {psnr_g:.2f} dB depth err {derr_g:.4f}")
    assert psnr_o > 15.0, "training did not converge enough for the comparison to mean anything"
    assert abs(psnr_g - psnr_o) < tol_db
    assert abs(derr_g - derr_o) < 0.1 * derr_o + 2e-3


def test_trained_psnr_20_objects_1000_steps():
    """SURVEY.md 8(c): identical-input 1000-step trajectory at the shipped shape (20 objects x 120 rays x 10 samples):
    trained PSNR of the fused tensor-core step within 0.2 dB of the oracle, object by object on average."""
    B, R, S, steps = 20, 120, 10, 1000
    params = vo.init_params(B, 32, seed=8)
    orc = vo.OracleEnsemble(params, 2.0)
    ens = make_ensemble(params, 2.0, 32, impl="umma")
    for it in range(steps):
        b = scene.sphere_batch(B, R, S, seed=5000 + it)
        orc.step(b)
        ens.step(to_dev(b))
    ens.check_status()
    held = scene.sphere_batch(B, 1000, S, seed=77)
    d_o, _, c_o, _ = orc.render(held)
    d_g, _, c_g, _ = ens.render(to_dev(held))
    psnr_o, derr_o = scene.quality(d_o, c_o, held)
    psnr_g, derr_g = scene.quality(d_g.cpu(), c_g.cpu(), held)
    print(f"[20 obj x 1000 steps] oracle PSNR {psnr_o:.2f} dB depth err {derr_o:.4f} | kernel PSNR {psnr_g:.2f} dB depth err {derr_g:.4f}")
    assert psnr_o > 15.0
    assert abs(psnr_g - psnr_o) < 0.2
    assert abs(derr_g - derr_o) < 0.1 * derr_o + 2e-3
