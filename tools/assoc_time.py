"""Per-frame time of ScanNet instance association on 620x460 synthetic frames (the shipped ScanNet crop), split into
classify / voxel / host hull / finalize, with the CPU numpy restatement of box_filter beside it (oracle/scannet_oracle,
which restates open3d with numpy / scipy: it is NOT open3d's time).

Run:  python tools/assoc_time.py [--frames 12] [--instances 20 40]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import scannet_oracle as so  # noqa: E402
from vmap_b200 import scannet  # noqa: E402
from vmap_b200.cfg import Config  # noqa: E402


def cfg_for(root):
    return Config(config_dict={
        "dataset": {"live": 0, "path": root, "format": "ScanNet", "keep_alive": 20},
        "optimizer": {"args": {"lr": 0.001, "weight_decay": 0.013}},
        "trainer": {"imap_mode": 0, "do_bg": 1, "n_models": 100, "train_device": "cuda:0", "data_device": "cuda:0",
                    "training_strategy": "vmap", "scale": 1000.0},
        "render": {"depth_range": [0.0, 6.0], "n_bins": 9, "n_bins_cam2surface": 1, "n_bins_cam2surface_bg": 5,
                   "iters_per_frame": 20, "n_per_optim": 120, "n_per_optim_bg": 1200},
        "model": {"n_unidir_funcs": 5, "obj_scale": 3.0, "bg_scale": 10.0, "surface_eps": 0.1, "other_eps": 0.05,
                  "keyframe_buffer_size": 20, "keyframe_step": 25, "keyframe_step_bg": 50, "window_size": 5,
                  "window_size_bg": 10, "hidden_feature_size": 32, "hidden_feature_size_bg": 128},
        "camera": {"w": 640, "h": 480, "mw": 10, "mh": 10},
        "vis": {"vis_device": "cuda:0", "n_vis_iter": 10000000, "grid_dim": 256, "live_voxel_size": 0.005},
    })


def run(n_inst, n_frames):
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=11, n_frames=n_frames, n_extra=max(n_inst - 7, 0), inf_frame=-1)
        ds = scannet.ScanNet(cfg_for(root))
        frames = [ds.decode(i) for i in range(n_frames)]
        tr = ds.trackers[0]
        ds.associate(frames[0])                      # warm-up: handle scratch, CUB temp storage
        tr.inst_dict.clear()
        tr.timing = True
        for k in tr.times:
            tr.times[k] = 0.0
        per_frame, split_frames = [], []
        for f in frames:                             # per-frame medians: the first frames carry one-off growth
            before = dict(tr.times)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ds.associate(f)
            torch.cuda.synchronize()
            per_frame.append(time.perf_counter() - t0)
            split_frames.append({k: tr.times[k] - before[k] for k in tr.times})
        gpu_total = float(np.median(per_frame))
        split = {k: float(np.median([s[k] for s in split_frames])) * 1e3 for k in tr.times}
        present = [len(np.unique(f[3])) for f in frames]
        seq = so.Sequence(root)
        cpu_frames = []
        for f in frames:
            color, depth, T, inst, sem = f
            t0 = time.perf_counter()
            labels = so.box_filter(inst, sem, depth, seq.tracks, seq.intr, np.linalg.inv(np.linalg.inv(T)))
            so.finalize(labels)
            cpu_frames.append(time.perf_counter() - t0)
        cpu = float(np.median(cpu_frames))
    return {"instances_per_frame": float(np.mean(present)), "gpu_median_ms_per_frame": gpu_total * 1e3,
            "split_ms": split, "cpu_numpy_restatement_median_ms_per_frame": cpu * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--instances", type=int, nargs="+", default=[20, 40])
    a = ap.parse_args()
    print("device:", torch.cuda.get_device_name(0))
    for n in a.instances:
        print(json.dumps({"target_instances": n, **run(n, a.frames)}))


if __name__ == "__main__":
    main()
