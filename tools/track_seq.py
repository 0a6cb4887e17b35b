"""Track a whole Replica-layout sequence on the GPU and score the trajectory against its ``traj_w_c.txt``.

    python tools/track_seq.py --config CFG --out DIR --slam [--frames a:b] [--n-iter N]
    python tools/track_seq.py --config CFG --out DIR --ckpt-dir LOG/ckpt --frame F [--frames a:b] [--n-iter N]

``--slam`` runs online SLAM (``vmap_b200.slam.Slam``): frame a takes its GT pose as the anchor, every later frame is
tracked against the map of the frames before it and then mapped from the tracked pose.  ``--ckpt-dir`` localises every
frame against the map of ``save_checkpoints`` files of frame F (loaded as ``tools/eval_2d.py`` loads them); frame a
starts from its GT pose, every later frame from the constant-velocity prediction of the two before it, never from GT.
Only the Replica layout (``rgb/``, ``depth/``, ``semantic_instance/``, ``semantic_class/``, ``traj_w_c.txt``) is read.

Writes ``traj_est.txt`` (``traj_w_c.txt`` format, one row per frame), ``metrics_traj.npy`` (a dict: ATE aligned and
unaligned, RPE, lost frames, per-frame device milliseconds) and prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from eval_2d import load_sources, replica_gt  # noqa: E402
from vmap_b200 import metrics  # noqa: E402
from vmap_b200.cfg import Config  # noqa: E402
from vmap_b200.slam import Slam  # noqa: E402

REPLICA_BACKGROUND_CLS = [5, 12, 30, 31, 40, 60, 92, 93, 95, 97, 98, 79]      # dataset.py:69
REPLICA_BBOX_SCALE = 0.2                                                     # dataset.py:72


def replica_frame(cfg, i):
    rgb, depth, T, inst = replica_gt(cfg, i)
    cls = cv2.imread(os.path.join(cfg.dataset_dir, "semantic_class", f"semantic_class_{i}.png"),
                     cv2.IMREAD_UNCHANGED).astype(np.int32).transpose(1, 0)
    return rgb, depth, T, inst, cls


def groups_from_sources(sources):
    by_ens = {}
    for s in sources:
        ent = by_ens.setdefault(id(s.ens), (s.ens, [None] * s.ens.n_obj))
        ent[1][s.row] = s.obj_id
    return list(by_ens.values())


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", required=True)
    ap.add_argument("--out", required=True)
    mode = ap.add_mutually_exclusive_group(required=True)
    mode.add_argument("--slam", action="store_true")
    mode.add_argument("--ckpt-dir")
    ap.add_argument("--frame", type=int, help="checkpoint frame (with --ckpt-dir)")
    ap.add_argument("--frames", default=None, help="a:b, the frames to run (default: all)")
    ap.add_argument("--n-iter", type=int, default=20, help="tracking iterations per frame")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--store-capacity", type=int, default=None,
                    help="initial frame-store slots (--slam; the store grows on demand)")
    args = ap.parse_args(argv)
    cfg = Config(args.config)
    if cfg.dataset_format != "Replica":
        raise SystemExit("track_seq.py reads the Replica layout only")
    if args.ckpt_dir and args.frame is None:
        raise SystemExit("--ckpt-dir needs --frame")
    os.makedirs(args.out, exist_ok=True)
    gt_all = np.loadtxt(os.path.join(cfg.dataset_dir, "traj_w_c.txt"), delimiter=" ").reshape(-1, 4, 4)
    n = len(os.listdir(os.path.join(cfg.dataset_dir, "depth")))
    a, b = 0, n
    if args.frames:
        lo, hi = args.frames.split(":")
        a, b = int(lo or 0), int(hi or n)
    frames = list(range(a, min(b, n)))
    kw = dict(n_track_iter=args.n_iter, seed=args.seed, background_cls=REPLICA_BACKGROUND_CLS,
              bbox_scale=REPLICA_BBOX_SCALE, max_frames=len(frames), timing=True,
              store_capacity=args.store_capacity)
    if args.slam:
        slam = Slam(cfg, T_init=gt_all[a], **kw)
    else:
        sources, skipped = load_sources(args.ckpt_dir, args.frame, device=cfg.data_device)
        if skipped:
            print("objects without a box in their checkpoint, not tracked:", skipped)
        slam = Slam(cfg, T_init=gt_all[a], map=False, groups=groups_from_sources(sources), **kw)
    for i in frames:
        rgb, depth, _, inst, cls = replica_frame(cfg, i)
        slam.step(torch.from_numpy(rgb), torch.from_numpy(depth), torch.from_numpy(inst), torch.from_numpy(cls))
    res = slam.result()
    times = slam.phase_times()
    est, gt = res["poses"], gt_all[frames]
    np.savetxt(os.path.join(args.out, "traj_est.txt"), est.reshape(-1, 16), delimiter=" ")
    out = {"mode": "slam" if args.slam else "localise", "frames": frames,
           "ate_aligned": metrics.ate(est, gt, align=True), "ate_unaligned": metrics.ate(est, gt, align=False),
           "rpe": metrics.rpe(est, gt) if len(frames) > 1 else None,
           "lost": [f for f, l in zip(frames, res["lost"]) if l], "times_ms": times,
           "tracked_ids": res["tracked_ids"], "inserted": res["inserted"], "track_modes": res["track_modes"]}
    np.save(os.path.join(args.out, "metrics_traj.npy"), np.array(out, dtype=object), allow_pickle=True)
    line = {"mode": out["mode"], "frames": len(frames), "ate_rmse_m": out["ate_aligned"]["rmse"],
            "ate_rmse_unaligned_m": out["ate_unaligned"]["rmse"],
            "rpe_trans_rmse_m": out["rpe"]["trans_rmse"] if out["rpe"] else None,
            "rpe_rot_rmse_deg": out["rpe"]["rot_rmse_deg"] if out["rpe"] else None,
            "lost": out["lost"], "frame_ms_median": float(np.median(times["frame"]))}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
