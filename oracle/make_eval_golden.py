"""Generate tests/golden/ref_metrics.npz: the reference's own metric/metrics.py (accuracy, completion, completion_ratio
at 1 cm and 5 cm, chamfer) on the seeded point sets of oracle/eval_oracle.METRIC_CASES.  Needs a reference checkout
(see oracle/_refload.py); no GPU.  Touches no other golden.

Run:  python -m oracle.make_eval_golden
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import _refload  # noqa: E402
from oracle import eval_oracle as eo  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_metrics.npz")


def ref_metrics():
    had = hasattr(np, "float")
    np.float = float                     # metric/metrics.py:7 uses the alias numpy >= 1.24 removed
    try:
        metrics = _refload.load("metric.metrics")
        out = {}
        for name, n_gt, n_rec, kind, seed in eo.METRIC_CASES:
            gt, rec = eo.metric_points(n_gt, n_rec, kind, seed)
            out[name + "_checksum"] = np.asarray([gt.sum(), rec.sum()], np.float64)    # guards the regenerated inputs
            out[name + "_accuracy"] = np.float64(metrics.accuracy(gt, rec))
            out[name + "_completion"] = np.float64(metrics.completion(gt, rec))
            out[name + "_ratio_0p01"] = np.float64(metrics.completion_ratio(gt, rec, 0.01))
            out[name + "_ratio_0p05"] = np.float64(metrics.completion_ratio(gt, rec, 0.05))
            out[name + "_chamfer"] = np.float64(metrics.chamfer(gt, rec))
        return out
    finally:
        if not had:
            del np.float


def main():
    np.savez_compressed(OUT, **ref_metrics())
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
