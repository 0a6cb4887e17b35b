"""GPU: the wgmma GEMMs (TMA-fed SWIZZLE_128B stages; generic tiled and weight-stationary kernels) of the
layer-wise wide-model path against torch.matmul, for the operand layouts / epilogues the path uses."""
import ctypes as C

import pytest
import torch

from vmap_b200 import _lib

pytestmark = pytest.mark.gpu


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def gemm(a_mn, b_mn, epi, M, N, K1, K2, a1, a2, b, bias=None, out16=None, out32=None, accumulate=0, ksplit=0, scale=1.0,
         ld32=None):
    L = _lib.lib()
    rc = L.vmb_debug_gemm(a_mn, b_mn, epi, M, N, K1, K2, _p(a1), a1.stride(0), _p(a2), a2.stride(0) if a2 is not None else 0,
                          _p(b), b.stride(0), _p(bias), _p(out16), out16.stride(0) if out16 is not None else 0,
                          _p(out32), (ld32 if ld32 else (out32.stride(0) if out32 is not None else 0)), accumulate, ksplit,
                          C.c_float(scale), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, L.vmb_last_error(None)
    torch.cuda.synchronize()


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def test_forward_layer_two_sources_bias_relu():
    torch.manual_seed(0)
    M, H = 300, 128
    x = (torch.randn(M, H, device="cuda") * 0.5).half()
    e = torch.randn(M, 144, device="cuda").half()                     # emb1 = first 96 columns of a 144-wide row
    w = (torch.randn(H, H + 96, device="cuda") * 0.1).half()
    bias = torch.randn(H, device="cuda")
    out = torch.zeros(M, H, device="cuda", dtype=torch.half)
    gemm(0, 0, 0, M, H, H, 96, x, e, w, bias=bias, out16=out)
    ref = torch.relu(torch.cat([x, e[:, :96]], 1).float() @ w.float().t() + bias)
    assert rel(out.float(), ref) < 2e-3


def test_ragged_n_and_fp32_store_accumulate():
    torch.manual_seed(1)
    M, N, K = 1000, 96, 256
    a = torch.randn(M, K, device="cuda").half()
    b = (torch.randn(N, K, device="cuda") * 0.1).half()
    out = torch.full((M, 144), 7.0, device="cuda")
    gemm(0, 0, 2, M, N, K, 0, a, None, b, out32=out[:, 10:], ld32=144, scale=0.5)
    ref = 0.5 * (a.float() @ b.float().t())
    assert rel(out[:, 10:106], ref) < 1e-3
    assert bool((out[:, :10] == 7.0).all()) and bool((out[:, 106:] == 7.0).all())
    gemm(0, 0, 2, M, N, K, 0, a, None, b, out32=out[:, 10:], ld32=144, accumulate=1, scale=0.5)
    assert rel(out[:, 10:106], 2 * ref) < 1e-3


def test_dgrad_mn_major_weight_view():
    """dX[:, j] = dY @ W[:, H + j]: B is the row-major weight matrix read as an MN-major operand."""
    torch.manual_seed(2)
    M, H = 700, 256
    dy = torch.randn(M, H, device="cuda").half()
    w = (torch.randn(H, H + 96, device="cuda") * 0.1).half()
    out = torch.zeros(M, 96, device="cuda")
    gemm(0, 1, 2, M, 96, H, 0, dy, None, w[:, H:], out32=out)
    assert rel(out, dy.float() @ w[:, H:].float()) < 1e-3
    out2 = torch.zeros(M, H, device="cuda")
    gemm(0, 1, 2, M, H, H, 0, dy, None, w[:, :H], out32=out2)
    assert rel(out2, dy.float() @ w[:, :H].float()) < 1e-3


def test_wgrad_split_k_atomics():
    """dW[o][k] = sum_p dY[p][o] X[p][k]: both operands MN-major, reduction over (ragged) points, split-K atomics."""
    torch.manual_seed(3)
    P, H = 1000, 128
    dy = (torch.randn(P, H, device="cuda") * 0.1).half()
    x = torch.randn(P, 144, device="cuda").half()
    g = torch.zeros(H, 100, device="cuda")
    gemm(1, 1, 3, H, 96, P, 0, dy, None, x, out32=g, ksplit=256, scale=2.0)
    ref = 2.0 * (dy.float().t() @ x[:, :96].float())
    assert rel(g[:, :96], ref) < 1e-3 and bool((g[:, 96:] == 0).all())


def test_throughput_wide_layer():
    M, H = 153600, 256
    x = torch.randn(M, H, device="cuda").half()
    e = torch.randn(M, 144, device="cuda").half()
    w = (torch.randn(H, H + 96, device="cuda") * 0.05).half()
    bias = torch.zeros(H, device="cuda")
    out = torch.empty(M, H, device="cuda", dtype=torch.half)
    for _ in range(3):
        gemm(0, 0, 0, M, H, H, 96, x, e, w, bias=bias, out16=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        gemm(0, 0, 0, M, H, H, 96, x, e, w, bias=bias, out16=out)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 100
    print(f"cat_layer-shaped GEMM {M}x{H}x{H + 96}: {us:.1f} us -> {2 * M * H * (H + 96) / us / 1e6:.1f} TFLOP/s")
    ref = torch.relu(torch.cat([x[:512], e[:512, :96]], 1).float() @ w.float().t())
    assert rel(out[:512].float(), ref) < 2e-3


WS = 16      # epi flag: weight-stationary kernel


@pytest.mark.parametrize("M,H,K2", [(1000, 128, 48), (300, 128, 96), (129, 64, 0), (5000, 256, 0)])
def test_ws_forward_layer(M, H, K2):
    torch.manual_seed(4)
    x = (torch.randn(M, H, device="cuda") * 0.5).half()
    e = torch.randn(M, 144, device="cuda").half()
    w = (torch.randn(H, H + K2, device="cuda") * 0.1).half()
    bias = torch.randn(H, device="cuda")
    out = torch.zeros(M, H, device="cuda", dtype=torch.half)
    gemm(0, 0, 0 | WS, M, H, H, K2, x, e if K2 else None, w, bias=bias, out16=out)
    ref = torch.relu(torch.cat([x, e[:, :K2]], 1).float() @ w.float().t() + bias)
    assert rel(out.float(), ref) < 2e-3


def test_ws_in_layer_k96():
    torch.manual_seed(5)
    M, H = 777, 256
    e = torch.randn(M, 144, device="cuda").half()
    w = (torch.randn(H, 96, device="cuda") * 0.1).half()
    bias = torch.randn(H, device="cuda")
    out = torch.zeros(M, H, device="cuda", dtype=torch.half)
    gemm(0, 0, 0 | WS, M, H, 96, 0, e, None, w, bias=bias, out16=out)
    assert rel(out.float(), torch.relu(e[:, :96].float() @ w.float().t() + bias)) < 2e-3


def test_ws_dgrad_mn_major_and_accumulate():
    torch.manual_seed(6)
    M, H = 700, 256
    dy = torch.randn(M, H, device="cuda").half()
    w = (torch.randn(H, H + 96, device="cuda") * 0.1).half()
    out = torch.full((M, 144), 3.0, device="cuda")
    gemm(0, 1, 2 | WS, M, 96, H, 0, dy, None, w[:, H:], out32=out, ld32=144)
    ref = dy.float() @ w[:, H:].float()
    assert rel(out[:, :96], ref) < 1e-3 and bool((out[:, 96:] == 3.0).all())
    gemm(0, 1, 2 | WS, M, 96, H, 0, dy, None, w[:, H:], out32=out, ld32=144, accumulate=1)
    assert rel(out[:, :96], 2 * ref) < 1e-3
    out2 = torch.zeros(M, H, device="cuda")
    gemm(0, 1, 2 | WS, M, H, H, 0, dy, None, w[:, :H], out32=out2)
    assert rel(out2, dy.float() @ w[:, :H].float()) < 1e-3
    out3 = torch.zeros(M, 48, device="cuda")
    gemm(0, 1, 2 | WS, M, 48, H, 0, dy, None, w[:, H:H + 48], out32=out3)
    assert rel(out3, dy.float() @ w[:, H:H + 48].float()) < 1e-3


def test_ws_throughput_hidden_layer():
    M, H = 153600, 256
    x = torch.randn(M, H, device="cuda").half()
    w = (torch.randn(H, H, device="cuda") * 0.05).half()
    bias = torch.zeros(H, device="cuda")
    out = torch.empty(M, H, device="cuda", dtype=torch.half)
    res = {}
    for name, flag in (("generic", 0), ("weight-stationary", WS)):
        for _ in range(3):
            gemm(0, 0, flag, M, H, H, 0, x, None, w, bias=bias, out16=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            gemm(0, 0, flag, M, H, H, 0, x, None, w, bias=bias, out16=out)
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 100
        res[name] = us
        print(f"hidden-layer GEMM {M}x{H}x{H} {name}: {us:.1f} us -> {2 * M * H * H / us / 1e6:.1f} TFLOP/s, "
              f"{(M * H * 4) / us / 1e3:.0f} GB/s in+out")
        assert rel(out[:512].float(), torch.relu(x[:512].float() @ w.float().t())) < 2e-3
