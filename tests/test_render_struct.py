"""CPU checks of the K9 view-rendering binding: argument struct in the header's field order, exports and limits."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    return open(os.path.join(ROOT, "include", "vmap_b200.h")).read()


def test_render_struct_matches_header_field_order():
    from vmap_b200 import _lib
    src = _header()
    body = src[src.index("typedef struct vmb_render_args"):src.index("} vmb_render_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"[\s\*]([a-z_0-9]+)\s*(?:\[\d+\])?\s*[;,]", body)
    assert names == [f[0] for f in _lib.RenderArgs._fields_]


def test_render_entry_points_and_limits():
    from vmap_b200 import _lib
    src = _header()
    for n in ("vmb_render_count", "vmb_render_emit", "vmb_render_composite"):
        assert n in _lib.EXPORTS and f"int {n}(" in src
    k = open(os.path.join(ROOT, "vmap_b200", "csrc", "k_render.cuh")).read()
    lim = dict(re.findall(r"#define (VMB_RENDER_[A-Z_]+) (\d+)", k))
    assert {n: int(v) for n, v in lim.items()} == {"VMB_RENDER_MAX_HITS": _lib.RENDER_MAX_HITS,
                                                  "VMB_RENDER_MAX_SRC": _lib.RENDER_MAX_SRC,
                                                  "VMB_RENDER_BOX": _lib.RENDER_BOX}
