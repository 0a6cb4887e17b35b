"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/vmap_b200.h declares, and its layout queries agree with the host mirror."""
import ctypes
import os
import re

import pytest

from vmap_b200 import _lib
from vmap_b200.layout import ALL_KEYS, host_offsets, tensor_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vmb_[a-z_]+)\s*\(", src)))


def test_header_symbols_are_all_bound_in_python():
    assert set(declared_symbols()) == set(_lib.EXPORTS)


def test_library_loads_and_exports_every_declared_symbol():
    if not os.path.isfile(_lib.LIB_PATH):
        _lib.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    for s in declared_symbols():
        assert hasattr(L, s), s
    assert b"sm_90a" in _lib.lib().vmb_version()


@pytest.mark.parametrize("hidden", [32, 64, 128, 256])
def test_param_layout_matches_host_mirror(hidden):
    if not os.path.isfile(_lib.LIB_PATH):
        _lib.build()
    count, stride, off, sz = _lib.param_layout(hidden, 6)
    assert (count, stride, off, sz) == host_offsets(hidden, 5)
    assert count == 4 * hidden * hidden + 225 * hidden + 4 + 63          # SURVEY.md 8a (a2) + PE
    assert stride % 32 == 0 and stride >= count
    shapes = tensor_shapes(hidden, 5)
    assert list(shapes) == list(ALL_KEYS)


def test_bad_arguments_return_error_codes_not_crashes():
    if not os.path.isfile(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    assert L.vmb_param_count(0, 6) < 0
    assert L.vmb_param_count(32, 99) < 0
    assert L.vmb_image_bytes(48, 6) == 0 and L.vmb_image_bytes(256, 6) == 2 * 256 * (4 * 256 + 240)
    assert L.vmb_step(None, None, None) < 0
    assert L.vmb_adam(None, None, None) < 0
    assert L.vmb_sample(None, None, None) < 0
    assert L.vmb_forward(None, None, None) < 0


def test_structs_match_header_field_order():
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    body = src[src.index("typedef struct vmb_step_args"):src.index("} vmb_step_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"[\s\*]([a-z_0-9]+)\s*[;,]", body)
    names = [n for n in names if n not in ("vmb_step_args",)]
    assert names == [f[0] for f in _lib.StepArgs._fields_]


def test_bench_product_arm_fails_loudly_without_gpu():
    """bench.py's product arm must never fall back to the CPU (the oracle is only the checker / the reference arm)."""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=300, cwd=root)
    assert r.returncode != 0 and "no CPU fallback" in (r.stdout + r.stderr)
    assert "{" not in r.stdout          # no JSON line, no number
