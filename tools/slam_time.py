"""Time the online SLAM loop per frame at the Replica vMAP shape and print one JSON line.

A synthetic sequence (``vmap_b200.synth.sphere_room_sequence``: 1200 x 680, 20 spheres as hidden-32 objects, the room
as the hidden-128 background, one sphere entering partway) runs through ``vmap_b200.slam.Slam`` with the shipped
Replica room0 vMAP settings: 20 tracking and 20 mapping iterations per frame.  CUDA events at the phase boundaries
give, per frame, the device time of the ingest (with the host read of the keep flags and boxes), the tracking, the
host bookkeeping the device waits for (keyframes, object insertion, sampler tables) and the mapping, and the whole
frame.  Medians are over the frames after the last object insertion; insertion frames (re-stack, graph captures) are
reported apart, and so is the tracking time of each tracking mode: a frame whose tracked set changed tracks eagerly,
the next frame with that set captures the tracking graph (a warm-up frame, a synchronise and the capture) and later
frames replay it.  The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from track_time import card  # noqa: E402
from vmap_b200 import metrics, synth  # noqa: E402
from vmap_b200.cfg import Config, replica_room0_dict  # noqa: E402
from vmap_b200.slam import Slam  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=40)
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "slam_time measures the GPU; there is no CPU number"
    cfg = Config(config_dict=replica_room0_dict())
    seq = synth.sphere_room_sequence(args.frames, cfg.W, cfg.H, cfg.fx, cfg.fy, cfg.cx, cfg.cy, n_extra=16)
    slam = Slam(cfg, T_init=seq["poses"][0], background_cls=seq["background_cls"], max_frames=args.frames,
                timing=True)
    for k in range(args.frames):
        slam.step(torch.from_numpy(seq["rgb"][k]), torch.from_numpy(seq["depth"][k].astype(np.float32)),
                  torch.from_numpy(seq["inst"][k]), torch.from_numpy(seq["cls"][k]))
    t = slam.phase_times()
    res = slam.result()
    last = max(res["inserted"].values())
    steady = list(range(last + 1, args.frames))
    ins = sorted(set(res["inserted"].values()))
    med = {k: round(float(np.median([v[i] for i in steady])), 3) for k, v in t.items()}
    ate = metrics.ate(res["poses"], seq["poses"])
    rpe = metrics.rpe(res["poses"], seq["poses"])
    out = {"card": card(), "shape": {"W": cfg.W, "H": cfg.H, "objects": len(slam.objects), "hidden": cfg.hidden_feature_size,
                                     "background_hidden": cfg.hidden_feature_size_bg, "track_iters": slam.n_track_iter,
                                     "map_iters": cfg.n_iter_per_frame, "frames": args.frames},
           "steady_frames": len(steady), "ms_median": med, "fps": round(1000.0 / med["frame"], 2),
           "insertion_frames": ins, "insertion_frame_ms": [round(t["frame"][i], 2) for i in ins],
           "track_ms_by_mode": {m: {"frames": len(v), "median": round(float(np.median(v)), 3)}
                                for m in ("eager", "capture", "replay")
                                for v in [[t["track"][i] for i, mm in enumerate(res["track_modes"]) if mm == m]] if v},
           "lost": int(res["lost"].sum()), "ate_rmse_m": ate["rmse"], "rpe_trans_rmse_m": rpe["trans_rmse"],
           "rpe_rot_rmse_deg": rpe["rot_rmse_deg"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
