"""Generate tests/golden/ref_scannet_{seq,workers}.npz: the reference's OWN dataset.ScanNet (dataset.py:150-292 with
utils.box_filter, utils.py:112-208) run on the seeded synthetic sequence of oracle/scannet_oracle.write_sequence.
Needs a reference checkout (see oracle/_refload.py); no GPU.  Touches no other golden.

open3d is replaced by the restated oracle/o3d_standin.py, ``np.int`` (removed in numpy 1.24, utils.py:114) is
shimmed to ``int``, and cv2.imshow / cv2.waitKey are no-ops.  Two goldens:
  seq      one dataset, frames in order (DataLoader with num_workers=0);
  workers  four datasets fed round-robin, frame i -> dataset i % 4 (the 4-worker DataLoader of dataset.py:49-55).
Goldens hold outputs only; tests regenerate the inputs from the seeded writer (PNG depth is lossless).

Run:  python -m oracle.make_scannet_golden
"""
from __future__ import annotations

import os
import sys
import tempfile
import types

import cv2
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import _refload  # noqa: E402
from oracle import o3d_standin  # noqa: E402
from oracle import scannet_oracle as so  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SEED, N_FRAMES = 3, 10


def ref_cfg(root):
    k = np.loadtxt(os.path.join(root, "intrinsic", "intrinsic_depth.txt"))
    return types.SimpleNamespace(imap_mode=0, dataset_dir=root, depth_scale=1 / 1000.0, max_depth=6.0, W=620, H=460,
                                 fx=k[0, 0], fy=k[1, 1], cx=k[0, 2] - 10, cy=k[1, 2] - 10, mw=10)


def pack(samples):
    """Per frame: obj [W, H], bbox_dict keys / rows, and every track of the dataset that made the frame."""
    out = {"n_frames": np.int64(len(samples))}
    for i, (smp, tracks) in enumerate(samples):
        out[f"obj_{i}"] = np.asarray(smp["obj"]).astype(np.int16)
        keys = sorted(smp["bbox_dict"])
        out[f"bbox_keys_{i}"] = np.asarray(keys, np.int64)
        out[f"bbox_{i}"] = np.stack([np.asarray(smp["bbox_dict"][k], np.int64).reshape(4) for k in keys])
        ids = sorted(tracks)
        out[f"track_ids_{i}"] = np.asarray(ids, np.int64)
        out[f"track_center_{i}"] = np.asarray([tracks[k][0] for k in ids], np.float64).reshape(-1, 3)
        out[f"track_R_{i}"] = np.asarray([tracks[k][1] for k in ids], np.float64).reshape(-1, 3, 3)
        out[f"track_extent_{i}"] = np.asarray([tracks[k][2] for k in ids], np.float64).reshape(-1, 3)
        out[f"track_npts_{i}"] = np.asarray([tracks[k][3] for k in ids], np.int64)
        out[f"track_cmp_{i}"] = np.asarray([tracks[k][4] for k in ids], np.int64)
    return out


def ref_run(root, n_workers):
    had_int = hasattr(np, "int")
    np.int = int
    prev = o3d_standin.install()
    show, wait = cv2.imshow, cv2.waitKey
    cv2.imshow, cv2.waitKey = (lambda *a, **k: None), (lambda *a, **k: -1)
    try:
        for n in ("utils", "dataset"):
            sys.modules.pop(n, None)
        dataset = _refload.load("dataset")
        cfg = ref_cfg(root)
        dss = [dataset.ScanNet(cfg) for _ in range(n_workers)]
        out = []
        for i in range(len(dss[0])):
            ds = dss[i % n_workers]
            smp = ds[i]
            tracks = {k: (np.asarray(t.bbox3D.center), np.asarray(t.bbox3D.R), np.asarray(t.bbox3D.extent),
                          len(t.pc.points), t.cmp_cnt) for k, t in ds.inst_dict.items()}
            out.append((smp, tracks))
        return out
    finally:
        cv2.imshow, cv2.waitKey = show, wait
        if prev is None:
            sys.modules.pop("open3d", None)
        else:
            sys.modules["open3d"] = prev
        if not had_int:
            del np.int
        for n in ("utils", "dataset"):
            sys.modules.pop(n, None)


def main():
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=SEED, n_frames=N_FRAMES)
        for name, nw in (("seq", 1), ("workers", 4)):
            path = os.path.join(GOLDEN, f"ref_scannet_{name}.npz")
            np.savez_compressed(path, seed=np.int64(SEED), **pack(ref_run(root, nw)))
            print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
