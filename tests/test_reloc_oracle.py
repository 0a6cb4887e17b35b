"""Relocalisation without a GPU: the hypothesis set, the selection order's restatement and the C declarations."""
import math
import os
import re

import numpy as np
import pytest

from vmap_b200 import reloc

HDR = os.path.join(os.path.dirname(__file__), "..", "include", "vmap_b200.h")


def select_order(scores, k):
    """vmb_reloc_select's order: finite scores ascending, ties to the lower index, then non-finite ones by index."""
    s = np.asarray(scores, np.float64)
    key = [(0, v, i) if np.isfinite(v) else (1, 0.0, i) for i, v in enumerate(s)]
    return [i for _, _, i in sorted(key)][:k]


@pytest.mark.parametrize("n,rot,trans", [(1, 30.0, 0.3), (17, 30.0, 0.3), (256, 45.0, 0.5), (4096, 7.5, 0.075)])
def test_hypotheses_deterministic_with_the_prior_and_within_the_spread(n, rot, trans):
    D = reloc.hypotheses(n, rot, trans)
    assert D.shape == (n, 4, 4) and D.dtype == np.float64
    assert np.array_equal(D, reloc._hypotheses.__wrapped__(n, rot, trans))
    assert np.array_equal(D[0], np.eye(4))
    R, t = D[:, :3, :3], D[:, :3, 3]
    assert np.abs(np.einsum("nij,nkj->nik", R, R) - np.eye(3)).max() < 1e-12
    assert np.abs(np.linalg.det(R) - 1.0).max() < 1e-12
    ang = np.degrees(np.arccos(np.clip((np.trace(R, axis1=1, axis2=2) - 1.0) / 2.0, -1.0, 1.0)))
    assert ang.max() <= rot + 1e-9 and np.linalg.norm(t, axis=1).max() <= trans + 1e-12
    assert np.all(D[:, 3] == [0.0, 0.0, 0.0, 1.0])
    if n >= 256:               # low discrepancy: the set fills its spread, not one corner of it
        assert ang.max() > 0.9 * rot and np.linalg.norm(t, axis=1).max() > 0.9 * trans
        assert len({tuple(np.round(x, 12)) for x in D.reshape(n, 16)}) == n


def test_hypotheses_reject_bad_arguments():
    for args in ((0, 10.0, 0.1), (4, -1.0, 0.1), (4, 10.0, float("nan"))):
        with pytest.raises(ValueError):
            reloc.hypotheses(*args)


def test_select_order_restatement():
    s = [3.0, 1.0, float("nan"), 1.0, -2.0, float("inf"), 0.5, -float("inf"), 1.0]
    assert select_order(s, 9) == [4, 6, 1, 3, 8, 0, 2, 5, 7]
    assert select_order(s, 3) == [4, 6, 1]


def test_declarations_match_the_binding():
    from vmap_b200 import _lib
    h = open(HDR).read()
    assert int(re.search(r"#define VMB_RELOC_MAX_HYP (\d+)", h).group(1)) == _lib.RELOC_MAX_HYP
    assert int(re.search(r"#define VMB_RELOC_MAX_K (\d+)", h).group(1)) == _lib.RELOC_MAX_K
    for name, n_args in (("vmb_reloc_score", 9), ("vmb_reloc_select", 8)):
        assert name in _lib.EXPORTS
        m = re.search(r"int " + name + r"\(([^)]*)\);", h, re.S)
        assert m and len(m.group(1).split(",")) == n_args, name
    src = open(reloc.__file__).read()
    assert "vmb_reloc_score(" in src and "vmb_reloc_select(" in src
    assert math.isclose(reloc.ROUND2_SHRINK, 0.25)
