"""Track a whole Replica- or ScanNet-layout sequence on the GPU and score the trajectory against its GT poses.

    python tools/track_seq.py --config CFG --out DIR --slam [--frames a:b] [--n-iter N] [--ba-every N --ba-iter M]
    python tools/track_seq.py --config CFG --out DIR --ckpt-dir LOG/ckpt --frame F [--frames a:b] [--n-iter N]

``--slam`` runs online SLAM (``vmap_b200.slam.Slam``): frame a takes its GT pose as the anchor, every later frame is
tracked against the map of the frames before it and then mapped from the tracked pose.  ``--ckpt-dir`` localises every
frame against the map of ``save_checkpoints`` files of frame F (loaded as ``tools/eval_2d.py`` loads them); frame a
starts from its GT pose, every later frame from the constant-velocity prediction of the two before it, never from GT.
Replica layout: ``rgb/``, ``depth/``, ``semantic_instance/``, ``semantic_class/`` and ``traj_w_c.txt``.  ScanNet layout
(``--slam`` only): every frame in order through ``scannet.read_sequence``; vMAP configs run with the instance
association (``Slam(assoc=...)``, one association state for the sequence), iMAP configs without.  The anchor is the
first frame of ``--frames`` with a finite GT pose (frames before it are not run); ATE and RPE are computed over the
frames whose GT pose is finite, and the others are listed as ``gt_invalid``.

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
from vmap_b200 import metrics, scannet  # noqa: E402
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
    ap.add_argument("--ba-every", type=int, default=0,
                    help="--slam: a bundle-adjustment pass after every N-th mapping frame (0: none)")
    ap.add_argument("--ba-iter", type=int, default=20, help="bundle-adjustment iterations per pass")
    ap.add_argument("--track-impl", choices=("fp32", "layerwise", "fused"), default=None,
                    help="tracking step (default: layerwise for iMAP configs, fp32 otherwise)")
    ap.add_argument("--ba-impl", choices=("fp32", "layerwise", "fused"), default=None,
                    help="bundle-adjustment step (default: layerwise for iMAP configs, fp32 otherwise)")
    args = ap.parse_args(argv)
    cfg = Config(args.config)
    if cfg.dataset_format not in ("Replica", "ScanNet"):
        raise SystemExit("track_seq.py reads the Replica and ScanNet layouts only")
    is_scannet = cfg.dataset_format == "ScanNet"
    if args.ckpt_dir and is_scannet:
        raise SystemExit("track_seq.py: --ckpt-dir (localisation against a saved map) reads Replica sequences only; "
                         "use --slam on ScanNet")
    if args.ckpt_dir and args.frame is None:
        raise SystemExit("--ckpt-dir needs --frame")
    os.makedirs(args.out, exist_ok=True)
    if is_scannet:
        gt_all = np.stack(scannet.ScanNet(cfg, n_trackers=0).poses)
    else:
        gt_all = np.loadtxt(os.path.join(cfg.dataset_dir, "traj_w_c.txt"), delimiter=" ").reshape(-1, 4, 4)
    n = len(os.listdir(os.path.join(cfg.dataset_dir, "depth")))
    a, b = 0, n
    if args.frames:
        lo, hi = args.frames.split(":")
        a, b = int(lo or 0), int(hi or n)
    frames = list(range(a, min(b, n)))
    if is_scannet:                                        # the anchor: the first frame with a finite GT pose
        finite = [i for i in frames if np.all(np.isfinite(gt_all[i]))]
        if not finite:
            raise SystemExit("track_seq.py: no frame in --frames has a finite GT pose to anchor the trajectory")
        frames = frames[frames.index(finite[0]):]
        a = frames[0]
    kw = dict(n_track_iter=args.n_iter, seed=args.seed, max_frames=len(frames), timing=True,
              store_capacity=args.store_capacity, track_impl=args.track_impl)
    if is_scannet:
        assoc = None
        if not cfg.imap_mode:
            assoc = scannet.InstanceTracker(cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.data_device,
                                            bbox_scale=scannet.BBOX_SCALE)
        kw.update(background_cls=[c for c in scannet.BG_CLASSES if c >= 0], bbox_scale=scannet.BBOX_SCALE,
                  assoc=assoc)
    else:
        kw.update(background_cls=REPLICA_BACKGROUND_CLS, bbox_scale=REPLICA_BBOX_SCALE)
    if args.slam:
        slam = Slam(cfg, T_init=gt_all[a], ba_every=args.ba_every, n_ba_iter=args.ba_iter, ba_impl=args.ba_impl, **kw)
    else:
        sources, skipped = load_sources(args.ckpt_dir, args.frame, device=cfg.data_device)
        if skipped:
            print("objects without a box in their checkpoint, not tracked:", skipped)
        slam = Slam(cfg, T_init=gt_all[a], map=False, groups=groups_from_sources(sources), **kw)
    if is_scannet:
        for f in scannet.read_sequence(cfg, frames):
            slam.step(f["rgb"], f["depth"], f["inst"], f["cls"])
    else:
        for i in frames:
            rgb, depth, _, inst, cls = replica_frame(cfg, i)
            slam.step(torch.from_numpy(rgb), torch.from_numpy(depth), torch.from_numpy(inst), torch.from_numpy(cls))
    res = slam.result()
    times = slam.phase_times()
    est, gt = res["poses"], gt_all[frames]
    np.savetxt(os.path.join(args.out, "traj_est.txt"), est.reshape(-1, 16), delimiter=" ")
    # ScanNet: score the frames with a finite GT pose only (metrics.ate / rpe with valid=)
    valid = np.ones(len(frames), bool) if is_scannet else None
    gt_ok = np.isfinite(gt.reshape(len(frames), -1)).all(1)
    has_pair = bool(np.any(gt_ok[:-1] & gt_ok[1:])) if len(frames) > 1 else False
    out = {"mode": "slam" if args.slam else "localise", "frames": frames,
           "ate_aligned": metrics.ate(est, gt, align=True, valid=valid),
           "ate_unaligned": metrics.ate(est, gt, align=False, valid=valid),
           "rpe": metrics.rpe(est, gt, valid=valid) if has_pair else None,
           "gt_invalid": [f for f, ok in zip(frames, gt_ok) if not ok],
           "lost": [f for f, l in zip(frames, res["lost"]) if l], "times_ms": times,
           "tracked_ids": res["tracked_ids"], "inserted": res["inserted"], "track_modes": res["track_modes"],
           "ba_loss": res["ba_loss"], "ba_frames": res["ba_frames"]}
    np.save(os.path.join(args.out, "metrics_traj.npy"), np.array(out, dtype=object), allow_pickle=True)
    line = {"mode": out["mode"], "frames": len(frames), "ate_rmse_m": out["ate_aligned"]["rmse"],
            "ate_rmse_unaligned_m": out["ate_unaligned"]["rmse"],
            "rpe_trans_rmse_m": out["rpe"]["trans_rmse"] if out["rpe"] else None,
            "rpe_rot_rmse_deg": out["rpe"]["rot_rmse_deg"] if out["rpe"] else None,
            "lost": out["lost"], "gt_invalid": out["gt_invalid"], "frame_ms_median": float(np.median(times["frame"])),
            "ba_passes": sum(1 for f in res["ba_frames"] if f)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
