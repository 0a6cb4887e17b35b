"""Time relocalisation scoring (vmb_reloc_score) at the Replica vMAP shape and print one JSON line.

20 hidden-32 objects x 120 rays x 10 samples on the fused tile: the scoring launch (forward, render, loss and the
ordered reduction) at H = 256 / 1024 / 4096 hypotheses, CUDA events over many launches, median [min, max] of three
timed windows; hypotheses per second; the tensor-core FLOPs of the forward from the wgmma shapes (K padded as the tile
runs them: (96 + 32 + 128 + 32 + 80) 32 + (32 + 32) 16 multiply-adds, 2 FLOP each, per point and hypothesis) and their share
of the H100 SXM dense fp16 data-sheet rate (989 TFLOP/s), with the card's name and power limit; and one whole
``Relocalizer.relocalise`` call (two scoring rounds of 256 x top 8, host clock around a synchronised call)."""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import vmap_oracle as vo  # noqa: E402
from vmap_b200.ensemble import VmapEnsemble  # noqa: E402
from vmap_b200.reloc import Relocalizer, hypotheses  # noqa: E402
from vmap_b200.track import SampleGroup  # noqa: E402

FP16_PEAK = 989e12
FLOP_PER_POINT = 2 * ((96 + 32 + 128 + 32 + 80) * 32 + (32 + 32) * 16)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip()


def main():
    assert torch.cuda.is_available(), "reloc_time needs a GPU"
    B, R, S = 20, 120, 10
    ens = VmapEnsemble(B, hidden=32, scale=2.0, device="cuda:0")
    ens.load_stacked(vo.init_params(B, 32, seed=0))
    sg = SampleGroup(ens, list(range(B)), vo.synthetic_batch(B, R, S, seed=1), 1, impl="fused")
    rl = Relocalizer([sg], n_hyp=256, top_k=8)
    out = {"card": card(), "shape": f"{B} objects x {R} rays x {S} samples, hidden 32", "score": {}}
    for H in (256, 1024, 4096):
        P = torch.from_numpy(hypotheses(H, 30.0, 0.3).copy()).cuda()
        for _ in range(3):
            rl.score(P)
        n = max(5, 20480 // H)
        runs = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                rl.score(P)
            e1.record()
            torch.cuda.synchronize()
            runs.append(e0.elapsed_time(e1) / n * 1e3)
        med = float(np.median(runs))
        flop = FLOP_PER_POINT * B * R * S * H
        out["score"][H] = {"us": [round(med, 1), round(min(runs), 1), round(max(runs), 1)],
                           "hyp_per_s": H / (med * 1e-6), "tflops": flop / (med * 1e-6) / 1e12,
                           "fp16_peak_share": flop / (med * 1e-6) / FP16_PEAK}
    prior = torch.eye(4, dtype=torch.float64, device="cuda:0")[None]
    for _ in range(3):
        rl.relocalise(prior)
    torch.cuda.synchronize()
    runs = []
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(10):
            rl.relocalise(prior)
        torch.cuda.synchronize()
        runs.append((time.perf_counter() - t0) / 10 * 1e3)
    out["relocalise_ms"] = [round(float(np.median(runs)), 3), round(min(runs), 3), round(max(runs), 3)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
