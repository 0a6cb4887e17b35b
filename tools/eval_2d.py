"""Render views of a trained map from its checkpoints and score them (the vMAP README's "2D Novel View Eval").

    python tools/eval_2d.py --config CFG --ckpt-dir LOG/ckpt --frame F --out DIR [--views 0,50,.. | --every N]
                            [--poses traj_w_c.txt] [--n-coarse 32 --n-fine 16]

Loads ``ckpt/{id}/obj_{id}_frame_{F}.pth`` (the format of sceneObject.save_checkpoints, vmap.py:461-476): the hidden
size comes from the FC_state_dict shapes, the scale from obj_scale, the box from bbox.  Objects of one hidden size
share one packed ensemble.  Checkpoints written by the reference pickle its top-level ``utils.BoundingBox``; that name
is mapped onto ``vmap_b200.utils.BoundingBox`` while unpickling.

Ground truth: Replica (``rgb/rgb_{i}.png``, ``depth/depth_{i}.png`` x depth_scale with depth above max_depth set to 0,
poses from ``traj_w_c.txt``, dataset.py:67-89,135) or ScanNet (``vmap_b200.scannet.ScanNet(cfg).decode(i)``).  Writes
``view_{i}_rgb.png``, ``view_{i}_depth.png`` (uint16 mm), ``view_{i}_inst.png`` (uint16, instance id + 1, 0 = none) and
``metrics_2D.npy`` (one dict per view), and prints the mean line.  With ``--poses`` the poses of that file are rendered
without ground truth (images only): the novel-trajectory case.
"""
from __future__ import annotations

import argparse
import glob
import os
import pickle
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from vmap_b200 import render, utils  # noqa: E402
from vmap_b200.cfg import Config  # noqa: E402
from vmap_b200.ensemble import VmapEnsemble  # noqa: E402
from vmap_b200.layout import FC_KEYS, PE_KEY  # noqa: E402
from vmap_b200.metrics import view_metrics  # noqa: E402


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if module == "utils" and name == "BoundingBox":        # the reference's top-level utils module
            return utils.BoundingBox
        return super().find_class(module, name)


_pickle_module = type(sys)("_eval2d_pickle")
_pickle_module.Unpickler = _Unpickler
_pickle_module.load = pickle.load


def load_checkpoint(path):
    return torch.load(path, map_location="cpu", weights_only=False, pickle_module=_pickle_module)


def load_sources(ckpt_dir: str, frame: int, device="cuda:0"):
    """Sources of every checkpoint of ``frame`` under ``ckpt_dir`` (one ensemble per hidden size)."""
    cks = []
    for d in sorted(glob.glob(os.path.join(ckpt_dir, "*"))):
        m = re.fullmatch(r"\d+", os.path.basename(d))
        f = os.path.join(d, f"obj_{os.path.basename(d)}_frame_{frame}.pth")
        if m and os.path.isfile(f):
            cks.append(load_checkpoint(f))
    cks.sort(key=lambda c: int(c["obj_id"]))
    by_hidden = {}
    for c in cks:
        by_hidden.setdefault(int(c["FC_state_dict"]["mid1.0.0.weight"].shape[0]), []).append(c)
    sources, skipped = [], []
    for hidden, group in by_hidden.items():
        # colour head input = hidden + emb_size2, emb_size2 = 21 * (n_freq) + 3 - 87 (trainer.py:16-17)
        n_freq = (group[0]["FC_state_dict"]["color_linear.0.weight"].shape[1] - hidden + 84) // 21
        ens = VmapEnsemble(len(group), hidden=hidden, n_unidir_funcs=n_freq - 1,
                           scale=[float(c["obj_scale"]) for c in group], device=device)
        ens.load_stacked({**{k: torch.stack([c["FC_state_dict"][k] for c in group]) for k in FC_KEYS},
                          PE_KEY: torch.stack([c["PE_state_dict"][PE_KEY] for c in group])})
        for row, c in enumerate(group):
            b = c["bbox"]
            if b is None:
                skipped.append(int(c["obj_id"]))
                continue
            bound_extent = 0.995 if int(c["obj_id"]) == 0 else 0.9          # trainer.py:33
            half = np.asarray(b.extent, np.float64) / (2.0 * bound_extent)
            sources.append(render.Source(ens, row, int(c["obj_id"]), np.asarray(b.center, np.float64),
                                         np.asarray(b.R, np.float64), half))
    sources.sort(key=lambda s: s.obj_id)
    return sources, skipped


def replica_gt(cfg, i):
    root = cfg.dataset_dir
    depth = cv2.imread(os.path.join(root, "depth", f"depth_{i}.png"), -1).astype(np.float32).transpose(1, 0)
    depth = depth * np.float32(cfg.depth_scale)
    depth[depth > cfg.max_depth] = 0.0
    rgb = cv2.cvtColor(cv2.imread(os.path.join(root, "rgb", f"rgb_{i}.png")), cv2.COLOR_BGR2RGB).transpose(1, 0, 2)
    T = np.loadtxt(os.path.join(root, "traj_w_c.txt"), delimiter=" ").reshape(-1, 4, 4)[i]
    inst_f = os.path.join(root, "semantic_instance", f"semantic_instance_{i}.png")
    inst = cv2.imread(inst_f, cv2.IMREAD_UNCHANGED).astype(np.int32).transpose(1, 0) if os.path.isfile(inst_f) else None
    return rgb, depth, T, inst


def scannet_gt(cfg, ds, i):
    dec = ds.decode(i)
    if dec is None:
        return None
    color, depth, T, inst, _ = dec
    return color.transpose(1, 0, 2), depth.transpose(1, 0), T, None if inst is None else inst.transpose(1, 0)


def write_view(out, i, img):
    col = (img["colour"].clamp(0, 1) * 255).round().to(torch.uint8).cpu().numpy().transpose(1, 0, 2)
    cv2.imwrite(os.path.join(out, f"view_{i}_rgb.png"), cv2.cvtColor(col, cv2.COLOR_RGB2BGR))
    dmm = (img["depth"] * 1000).round().clamp(0, 65535).to(torch.int32).cpu().numpy().astype(np.uint16).T
    cv2.imwrite(os.path.join(out, f"view_{i}_depth.png"), dmm)
    inst = (img["instance"] + 1).clamp(0, 65535).cpu().numpy().astype(np.uint16).T
    cv2.imwrite(os.path.join(out, f"view_{i}_inst.png"), inst)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", required=True)
    ap.add_argument("--ckpt-dir", required=True)
    ap.add_argument("--frame", type=int, required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--views", default=None, help="comma-separated frame indices")
    ap.add_argument("--every", type=int, default=None)
    ap.add_argument("--poses", default=None, help="traj_w_c.txt-format poses to render without ground truth")
    ap.add_argument("--n-coarse", type=int, default=32)
    ap.add_argument("--n-fine", type=int, default=16)
    args = ap.parse_args(argv)
    cfg = Config(args.config)
    os.makedirs(args.out, exist_ok=True)
    sources, skipped = load_sources(args.ckpt_dir, args.frame)
    if skipped:
        print("objects without a box, not rendered:", skipped)
    K = np.array([[cfg.fx, 0, cfg.cx], [0, cfg.fy, cfg.cy], [0, 0, 1.0]])
    kw = dict(n_coarse=args.n_coarse, n_fine=args.n_fine, surface_eps=cfg.surface_eps, near=cfg.min_depth,
              far=cfg.max_depth)
    if args.poses:
        poses = np.loadtxt(args.poses, delimiter=" ").reshape(-1, 4, 4)
        views = range(len(poses)) if args.views is None else [int(v) for v in args.views.split(",")]
        for i in views[::args.every or 1]:
            img, _ = render.render_view(sources, poses[i], K, cfg.W, cfg.H, **kw)
            write_view(args.out, i, img)
        print(f"rendered {len(views[::args.every or 1])} poses to {args.out}")
        return
    scannet = cfg.dataset_format != "Replica"
    if scannet:
        from vmap_b200.scannet import ScanNet
        ds = ScanNet(cfg)
        n = len(ds)
    else:
        n = len(os.listdir(os.path.join(cfg.dataset_dir, "depth")))
    views = [int(v) for v in args.views.split(",")] if args.views else list(range(0, n, args.every or 1))
    results = []
    for i in views:
        gt = scannet_gt(cfg, ds, i) if scannet else replica_gt(cfg, i)
        if gt is None:
            continue
        rgb, depth, T, inst = gt
        img, stats = render.render_view(sources, T, K, cfg.W, cfg.H, **kw)
        write_view(args.out, i, img)
        m = view_metrics(img["colour"], img["depth"], torch.from_numpy(rgb.astype(np.float32) / 255.0),
                         torch.from_numpy(depth), None if inst is None else torch.from_numpy(inst))
        m.update(view=i, **stats)
        results.append(m)
    np.save(os.path.join(args.out, "metrics_2D.npy"), np.array(results, dtype=object), allow_pickle=True)
    keys = [k for k in ("psnr", "depth_l1", "obj_psnr") if results and k in results[0]]
    print("mean over %d views: " % len(results) + ", ".join(f"{k} {np.mean([r[k] for r in results]):.4f}" for k in keys))


if __name__ == "__main__":
    main()
