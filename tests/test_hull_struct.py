"""CPU checks of the K8 convex-hull / box bindings: argument structs in the header's field order."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("c_name,py_name", [("vmb_hull_args", "HullArgs"), ("vmb_obb_args", "ObbArgs")])
def test_hull_structs_match_header_field_order(c_name, py_name):
    from vmap_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    body = src[src.index("typedef struct " + c_name):src.index("} " + c_name + ";")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"[\s\*]([a-z_0-9]+)\s*(?:\[\d+\])?\s*[;,]", body)
    assert names == [f[0] for f in getattr(_lib, py_name)._fields_]


def test_hull_entry_points_and_status_codes():
    from vmap_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    for n in ("vmb_hull", "vmb_obb_minvol"):
        assert n in _lib.EXPORTS and f"int {n}(" in src
    codes = dict(re.findall(r"(VMB_HULL_[A-Z_]+) = (\d+)", src))
    assert {k: int(v) for k, v in codes.items()} == {"VMB_HULL_OK": _lib.HULL_OK, "VMB_HULL_TOO_FEW": _lib.HULL_TOO_FEW,
                                                     "VMB_HULL_FLAT": _lib.HULL_FLAT, "VMB_HULL_BAD": _lib.HULL_BAD}
