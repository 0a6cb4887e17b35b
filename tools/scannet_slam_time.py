"""Time online SLAM per frame at the ScanNet vMAP shape, with the instance association, and print one JSON line.

A synthetic sequence (``vmap_b200.synth.sphere_room_sequence`` written by ``synth.write_scannet``: 620 x 460 after the
10-pixel edge crop, 20 spheres as hidden-32 objects, the room as the hidden-128 background, one sphere entering partway)
is read back through ``scannet.read_sequence`` and runs through ``vmap_b200.slam.Slam(assoc=...)`` with the shipped
ScanNet vMAP settings (``do_bg``, 20 tracking and 20 mapping iterations per frame).  CUDA events at the phase boundaries
give, per frame, the device time of the ingest, the tracking, the association (with the relabel and its table read),
the host bookkeeping and the mapping.  Medians are over the frames after the last object insertion.  A second run with
``InstanceTracker.timing`` (which synchronises after every stage) splits the association into classify / voxel /
hull / finalize.  ``--min-pixels``: the association's eroded-pixel threshold for a new id (the reference's 1500 keeps
the smaller spheres out of the map at this size).  The card's name, power limit and maximum SM clock are read in the
same run."""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from track_time import card  # noqa: E402
from vmap_b200 import metrics, scannet, synth  # noqa: E402
from vmap_b200.cfg import Config  # noqa: E402
from vmap_b200.slam import Slam  # noqa: E402

W, H, MW, FX = 620, 460, 10, 577.87          # ScanNet's 640 x 480 depth camera, cropped by 10 px


def scannet_vmap_dict(path: str) -> dict:
    """The shipped ScanNet vMAP settings (config_scannet0000_vMAP.json) with the dataset at ``path``."""
    return {
        "dataset": {"live": 0, "path": path, "format": "ScanNet", "keep_alive": 20},
        "optimizer": {"args": {"lr": 0.001, "weight_decay": 0.013, "pose_lr": 0.001}},
        "trainer": {"imap_mode": 0, "do_bg": 1, "n_models": 100, "train_device": "cuda:0", "data_device": "cuda:0",
                    "training_strategy": "vmap", "epochs": 1000000, "scale": 1000.0},
        "render": {"depth_range": [0.0, 6.0], "n_bins": 9, "n_bins_cam2surface": 1, "n_bins_cam2surface_bg": 5,
                   "iters_per_frame": 20, "n_per_optim": 120, "n_per_optim_bg": 1200},
        "model": {"n_unidir_funcs": 5, "obj_scale": 3.0, "bg_scale": 10.0, "color_scaling": 5.0,
                  "opacity_scaling": 10.0, "gt_scene": 1, "surface_eps": 0.1, "other_eps": 0.05,
                  "keyframe_buffer_size": 20, "keyframe_step": 25, "keyframe_step_bg": 50, "window_size": 5,
                  "window_size_bg": 10, "hidden_layers_block": 1, "hidden_feature_size": 32,
                  "hidden_feature_size_bg": 128},
        "camera": {"w": W + 2 * MW, "h": H + 2 * MW, "mw": MW, "mh": MW},
        "vis": {"vis_device": "cuda:0", "n_vis_iter": 10000000, "n_bins_fine_vis": 10, "im_vis_reduce": 10,
                "grid_dim": 256, "live_vis": 1, "live_voxel_size": 0.005},
    }


def run(cfg, frames, min_pixels, split=False):
    torch.manual_seed(0)
    random.seed(0)
    tracker = scannet.InstanceTracker(cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.data_device, min_pixels=min_pixels,
                                      bbox_scale=scannet.BBOX_SCALE)
    tracker.timing = split
    slam = Slam(cfg, T_init=frames[0]["T"], assoc=tracker, max_frames=len(frames), timing=not split)
    for f in frames:
        slam.step(f["rgb"], f["depth"], f["inst"], f["cls"])
    torch.cuda.synchronize()
    return slam, tracker


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--min-pixels", type=int, default=400)
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "scannet_slam_time measures the GPU; there is no CPU number"
    seq = synth.sphere_room_sequence(args.frames, W, H, FX, FX, W / 2 - 0.5, H / 2 - 0.5, n_extra=16)
    with tempfile.TemporaryDirectory() as root:
        synth.write_scannet(root, seq, mw=MW)
        cfg = Config(config_dict=scannet_vmap_dict(root))
        frames = list(scannet.read_sequence(cfg))
    slam, _ = run(cfg, frames, args.min_pixels)
    t = slam.phase_times()
    res = slam.result()
    last = max(res["inserted"].values())
    steady = list(range(last + 1, args.frames))
    med = {k: round(float(np.median([v[i] for i in steady])), 3) for k, v in t.items()}
    _, tr = run(cfg, frames, args.min_pixels, split=True)
    split = {k: round(1000.0 * v / args.frames, 3) for k, v in tr.times.items()}
    ate = metrics.ate(res["poses"], seq["poses"])
    rpe = metrics.rpe(res["poses"], seq["poses"])
    out = {"card": card(), "shape": {"W": cfg.W, "H": cfg.H, "objects": len(slam.objects), "do_bg": cfg.do_bg,
                                     "track_iters": slam.n_track_iter, "map_iters": cfg.n_iter_per_frame,
                                     "frames": args.frames, "min_pixels": args.min_pixels},
           "steady_frames": len(steady), "ms_median": med, "fps": round(1000.0 / med["frame"], 2),
           "assoc_split_ms_per_frame": split, "lost": int(res["lost"].sum()), "ate_rmse_m": ate["rmse"],
           "rpe_trans_rmse_m": rpe["trans_rmse"], "rpe_rot_rmse_deg": rpe["rot_rmse_deg"],
           "track_impl": slam.track_kw["impl"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
