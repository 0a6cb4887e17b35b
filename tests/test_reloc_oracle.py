"""Relocalisation without a GPU: the hypothesis set, the selection order's restatement and the C declarations."""
import contextlib
import math
import os
import re

import numpy as np
import pytest
import torch

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


def test_select_order_all_non_finite_infinities_and_signed_zeros():
    nan, inf = float("nan"), float("inf")
    assert select_order([nan] * 5, 5) == [0, 1, 2, 3, 4]
    assert select_order([inf, -inf, 2.0, nan, -inf, -1.0], 6) == [5, 2, 0, 1, 3, 4]
    assert select_order([0.0, -0.0, 1.0, -0.0, 0.0, -1.0], 6) == [5, 0, 1, 3, 4, 2]
    assert select_order([7.0], 1) == [0]


# ---- Relocalizer's argument checks, on a stand-in group whose library must never be reached ------------------------

class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


class _Ens:
    device, hidden, colour_scaling, opacity_scaling = torch.device("cpu"), 32, 5.0, 10.0
    lib, image, _handle = _NoLaunch(), None, None

    def _on_device(self):
        return contextlib.nullcontext()


class _Group:
    path, ens, active = "fused", _Ens(), [0, 1, 2]

    def bind(self, g, it):
        pass


def _reloc(n_groups=1):
    return reloc.Relocalizer([_Group() for _ in range(n_groups)], n_hyp=16, top_k=4)


def test_score_checks_its_arguments_before_any_launch():
    from vmap_b200 import _lib
    rl = _reloc()
    P = torch.eye(4, dtype=torch.float64).repeat(6, 1, 1)
    f64 = dict(dtype=torch.float64)
    bad = [(P[:, :, :3], None), (P.reshape(6, 16), None), (P.reshape(2, 3, 4, 4), None), (P.long(), None),
           (P[:0], None), (P[:1].expand(_lib.RELOC_MAX_HYP + 1, 4, 4), None), (P.numpy(), None),
           (P, torch.zeros(6, 3, 4)), (P, torch.zeros(6, 2, 4, **f64)), (P, torch.zeros(5, 3, 4, **f64)),
           (P, torch.zeros(6, 3, 5, **f64)), (P, torch.zeros(4, 3, 6, **f64).permute(2, 1, 0)),
           (P, torch.zeros(72, **f64)), (P, np.zeros((6, 3, 4)))]
    for poses, terms in bad:
        with pytest.raises(_lib.VmbError):
            rl.score(poses, terms)
    with pytest.raises(_lib.VmbError, match="one group"):       # one buffer of terms cannot hold two groups' rows
        _reloc(2).score(P, torch.zeros(6, 3, 4, **f64))
    for poses, terms in ((P, None), (P[0], None), (P, torch.zeros(6, 3, 4, **f64)), (P.float(), None)):
        with pytest.raises(AssertionError, match="vmb_reloc_score"):   # well-formed: they reach the library
            rl.score(poses, terms)


def test_select_checks_its_arguments_before_any_launch():
    from vmap_b200 import _lib
    rl = _reloc()
    s = torch.arange(6, dtype=torch.float64)
    P = torch.eye(4, dtype=torch.float64).repeat(6, 1, 1)
    big = _lib.RELOC_MAX_HYP + 1
    bad = [(s.float(), P, 2), (s[None], P, 2), (s[:0], P[:0], 1), (s.numpy(), P, 2), (s, P[:5], 2), (s, P.float(), 2),
           (s, P.reshape(6, 16), 2), (s, P.numpy(), 2), (s, P, 0), (s, P, 7), (s, P, 2.5), (s, P, True),
           (torch.zeros(big, dtype=torch.float64), torch.zeros(big, 4, 4, dtype=torch.float64), 2),
           (torch.zeros(100, dtype=torch.float64), torch.zeros(100, 4, 4, dtype=torch.float64), _lib.RELOC_MAX_K + 1)]
    for scores, poses, k in bad:
        with pytest.raises(_lib.VmbError):
            rl.select(scores, poses, k)
    for k in (1, 6):
        with pytest.raises(AssertionError, match="vmb_reloc_select"):
            rl.select(s, P, k)
