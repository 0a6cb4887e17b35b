"""Time iMAP (``--mode imap``, the default) or vMAP (``--mode vmap``) mapping and SLAM with and without joint keyframe
poses and print one JSON line.

A synthetic sequence at the iMAP shape (``vmap_b200.synth.sphere_room_sequence``, 1200 x 680; the shipped iMAP
settings: one hidden-256 scene model, ``n_per_optim`` 4800 rays of 5 + 9 bins, 20 mapping and 20 tracking iterations per
frame) runs through ``vmap_b200.slam.Slam`` with graphs on, once with ``joint_poses=False`` and once with
``joint_poses=True``, alternating, three times each.  CUDA events at the phase boundaries give per frame the device
time of the mapping frame (graph replay once the object set is stable) and of the whole frame; each run reports the
medians over its frames after the first two (insertion, graph captures), and the JSON line gives median [min, max] over
the three runs, with frames/s from the frame medians.  Then one joint mapping frame runs eagerly under
``torch.profiler`` (CUDA activities) for the device time per launch of the kernels the joint mode adds
(``k_joint_world``, ``k_tlw_pose``, ``k_tlw_reduce``) and of the pose update (``k_ba_update``).  The card's name, power
limit and max SM clock are read in the same run.

``--mode vmap``: the Replica vMAP shape (1200 x 680; 4 + 16 spheres, so 20 hidden-32 objects of 120 rays per
iteration, and the hidden-128 background of 1200 rays per iteration, 20 iterations) with ``joint_impl="fused"``.  The
profiled frame is taken in both modes, so the fused step's JOINT and plain instantiations are both timed; the JSON line
also gives ``k_joint_rows`` and the rest of the frame's kernels (the background's joint step and the samplers)."""
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

KERNELS = ("k_joint_world", "k_tlw_pose", "k_tlw_reduce", "k_ba_update")
KERNELS_VMAP = ("k_joint_world", "k_step_fused", "k_joint_rows", "k_tlw_pose", "k_tlw_reduce", "k_ba_update")


def run(cfg, seq, frames: int, joint: bool, vmap: bool = False):
    kw = dict(joint_impl="fused", background_cls=seq["background_cls"]) if vmap and joint else \
        dict(background_cls=seq["background_cls"]) if vmap else {}
    slam = Slam(cfg, T_init=seq["poses"][0], max_frames=frames, timing=True, joint_poses=joint, **kw)
    for k in range(frames):
        inst = (torch.from_numpy(seq["inst"][k]), torch.from_numpy(seq["cls"][k])) if vmap else (None,)
        slam.step(torch.from_numpy(seq["rgb"][k]), torch.from_numpy(seq["depth"][k].astype(np.float32)), *inst)
    t = slam.phase_times()
    res = slam.result()
    steady = range(2, frames)
    return (float(np.median([t["map"][i] for i in steady])), float(np.median([t["frame"][i] for i in steady])),
            metrics.ate(res["poses"], seq["poses"][:frames])["rmse"], int(res["lost"].sum()), slam)


def kernel_ms(slam, kernels=KERNELS) -> dict:
    """Device time per launch of the joint mode's added kernels and the pose update, from one eager mapping frame."""
    from torch.profiler import ProfilerActivity, profile
    loop = slam.loop
    loop._enqueue(upload=False)                     # warm (the tables of the last frame are already on the device)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loop._enqueue(upload=False)
        torch.cuda.synchronize()
    out, total, named = {}, 0.0, 0.0
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total += us
        for k in kernels:
            if k in ev.key:
                key = k
                if k == "k_step_fused":          # the JOINT instantiation or the plain one
                    key += "_joint" if "true" in ev.key else "_plain"
                out[key] = {"launches": ev.count, "us_per_launch": round(us / max(ev.count, 1), 2)}
                named += us
                break
    out["all_kernels_ms_per_frame"] = round(total / 1000.0, 3)
    if kernels is not KERNELS:
        out["other_kernels_ms_per_frame"] = round((total - named) / 1000.0, 3)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--mode", choices=("imap", "vmap"), default="imap")
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "joint_time measures the GPU; there is no CPU number"
    vmap = args.mode == "vmap"
    cfg = Config(config_dict=replica_room0_dict(imap=not vmap))
    seq = synth.sphere_room_sequence(args.frames, cfg.W, cfg.H, cfg.fx, cfg.fy, cfg.cx, cfg.cy,
                                     n_extra=16 if vmap else 0)
    rec = {False: [], True: []}
    last = last_plain = None
    for _ in range(args.runs):
        for joint in (False, True):
            r = run(cfg, seq, args.frames, joint, vmap)
            rec[joint].append(r[:4])
            last = r[4] if joint else last
            last_plain = r[4] if not joint else last_plain

    def stat(xs, f=lambda v: v):
        v = [f(x) for x in xs]
        return [round(float(np.median(v)), 3), round(float(min(v)), 3), round(float(max(v)), 3)]

    out = {"card": card(), "shape": {"W": cfg.W, "H": cfg.H, "hidden": cfg.hidden_feature_size,
                                     "n_per_optim": cfg.n_per_optim, "bins": [cfg.n_bins_cam2surface, cfg.n_bins],
                                     "map_iters": cfg.n_iter_per_frame, "frames": args.frames, "runs": args.runs},
           "stat": "median [min, max] over runs of the per-run median over frames 2..",
           "map_frame_ms": {"plain": stat([r[0] for r in rec[False]]), "joint": stat([r[0] for r in rec[True]])},
           "frame_ms": {"plain": stat([r[1] for r in rec[False]]), "joint": stat([r[1] for r in rec[True]])},
           "slam_fps": {"plain": stat([r[1] for r in rec[False]], lambda v: 1000.0 / v),
                        "joint": stat([r[1] for r in rec[True]], lambda v: 1000.0 / v)},
           "ate_rmse_cm": {"plain": stat([r[2] * 100 for r in rec[False]]),
                           "joint": stat([r[2] * 100 for r in rec[True]])},
           "lost": {"plain": sum(r[3] for r in rec[False]), "joint": sum(r[3] for r in rec[True])}}
    out["map_frame_ratio"] = round(out["map_frame_ms"]["joint"][0] / out["map_frame_ms"]["plain"][0], 3)
    if vmap:
        out["mode"] = "vmap"
        out["shape"].update(hidden=cfg.hidden_feature_size, hidden_bg=cfg.hidden_feature_size_bg,
                            n_obj=last.ens.n_obj, rays_per_iter=cfg.n_samples_per_frame * cfg.win_size,
                            rays_per_iter_bg=cfg.n_samples_per_frame_bg * cfg.win_size_bg)
        out["joint_kernels"] = kernel_ms(last, KERNELS_VMAP)
        out["plain_kernels"] = kernel_ms(last_plain, KERNELS_VMAP)
    else:
        out["joint_kernels"] = kernel_ms(last)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
