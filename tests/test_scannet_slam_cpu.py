"""CPU checks for SLAM on ScanNet sequences: the sphere room written in the ScanNet layout reads back through the
restated loader, trajectory metrics over the frames with a valid GT pose, the SLAM-side reader, and the relabel
binding against the header."""
import os
import re

import numpy as np
import pytest

from oracle import scannet_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, FX, MW = 96, 72, 72.0, 6


@pytest.fixture(scope="module")
def seq():
    from vmap_b200 import synth
    return synth.sphere_room_sequence(5, W, H, FX, FX, W / 2 - 0.5, H / 2 - 0.5)


def test_write_scannet_round_trip(seq, tmp_path):
    from vmap_b200 import synth
    root = str(tmp_path)
    synth.write_scannet(root, seq, mw=MW, inf_frames=(2,))
    poses = so.load_poses(root)
    assert len(poses) == 5
    for i in range(5):
        if i == 2:
            assert np.all(np.isinf(poses[i]))
            continue
        assert np.array_equal(poses[i], seq["poses"][i])
        # the restated loader skips inf poses; frame i is read as itself when its own pose is finite
        color, depth, T, inst, sem = so.load_frame(root, i, W, H, MW, 1 / 1000.0, 100.0, poses)
        assert color.shape == (H, W, 3) and depth.shape == (H, W)
        assert np.array_equal(T, seq["poses"][i])
        assert np.abs(depth.T.astype(np.float64) - seq["depth"][i]).max() <= 1e-3 * (1 + 1e-6)
        np.testing.assert_array_equal(inst.T, seq["inst"][i])
        np.testing.assert_array_equal(sem.T.astype(np.int32), synth.scannet_classes(seq["inst"][i]))
    # the intrinsics the config reads give back the test camera after the crop
    seqr = so.Sequence(root, W=W, H=H, edge=MW)
    assert seqr.intr == (FX, FX, W / 2 - 0.5, H / 2 - 0.5)
    # spheres carry a class that is not background, the room's planes one that is
    cls = synth.scannet_classes(seq["inst"][0])
    assert not np.isin(cls[seq["inst"][0] < 20], so.BG_CLASSES).any()
    assert np.isin(cls[seq["inst"][0] >= 20], so.BG_CLASSES).all()


def _scannet_cfg(root, imap=False):
    from vmap_b200.cfg import Config
    d = {
        "dataset": {"live": 0, "path": root, "format": "ScanNet", "keep_alive": 20},
        "optimizer": {"args": {"lr": 0.001, "weight_decay": 0.013, "pose_lr": 0.001}},
        "trainer": {"imap_mode": int(imap), "do_bg": 0, "n_models": 100, "train_device": "cuda:0",
                    "data_device": "cuda:0", "training_strategy": "vmap", "epochs": 1000000, "scale": 1000.0},
        "render": {"depth_range": [0.0, 100.0], "n_bins": 9, "n_bins_cam2surface": 1, "n_bins_cam2surface_bg": 5,
                   "iters_per_frame": 20, "n_per_optim": 120, "n_per_optim_bg": 1200},
        "model": {"n_unidir_funcs": 5, "obj_scale": 2.0, "bg_scale": 5.0, "color_scaling": 5.0,
                  "opacity_scaling": 10.0, "gt_scene": 1, "surface_eps": 0.1, "other_eps": 0.05,
                  "keyframe_buffer_size": 20, "keyframe_step": 25, "keyframe_step_bg": 50, "window_size": 5,
                  "window_size_bg": 10, "hidden_layers_block": 1, "hidden_feature_size": 32,
                  "hidden_feature_size_bg": 128},
        "camera": {"w": W + 2 * MW, "h": H + 2 * MW, "mw": MW, "mh": MW},
        "vis": {"vis_device": "cuda:0", "n_vis_iter": 10000000, "n_bins_fine_vis": 10, "im_vis_reduce": 10,
                "grid_dim": 256, "live_vis": 1, "live_voxel_size": 0.005},
    }
    return Config(config_dict=d)


@pytest.mark.parametrize("imap", [False, True])
def test_read_sequence_yields_every_frame_in_order(seq, tmp_path, imap):
    from vmap_b200 import scannet, synth
    root = str(tmp_path)
    synth.write_scannet(root, seq, mw=MW, inf_frames=(2,))
    cfg = _scannet_cfg(root, imap)
    assert (cfg.W, cfg.H, cfg.fx, cfg.cx) == (W, H, FX, W / 2 - 0.5)
    out = list(scannet.read_sequence(cfg, prefetch=2))
    assert [f["index"] for f in out] == list(range(5))
    for i, f in enumerate(out):
        assert f["rgb"].shape == (W, H, 3) and f["depth"].shape == (W, H)
        assert np.all(np.isinf(f["T"])) if i == 2 else np.array_equal(f["T"], seq["poses"][i])
        if imap:
            assert f["inst"] is None and f["cls"] is None
        else:
            np.testing.assert_array_equal(f["inst"].numpy(), seq["inst"][i])
            np.testing.assert_array_equal(f["cls"].numpy(), synth.scannet_classes(seq["inst"][i]))
    sub = list(scannet.read_sequence(cfg, frames=[3, 1], prefetch=0))
    assert [f["index"] for f in sub] == [3, 1]


def _trajectory(n, seed):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    T = np.tile(np.eye(4), (n, 1, 1))
    T[:, :3, :3] = Rotation.from_rotvec(rng.normal(0, 0.3, (n, 3))).as_matrix()
    T[:, :3, 3] = rng.normal(0, 1.0, (n, 3))
    return T


def test_trajectory_metrics_over_valid_frames():
    from vmap_b200 import metrics
    n = 12
    gt, est = _trajectory(n, 1), _trajectory(n, 2)
    # valid=None and an all-True mask are today's metrics
    for align in (True, False):
        a, b = metrics.ate(est, gt, align=align), metrics.ate(est, gt, align=align, valid=np.ones(n, bool))
        assert a["rmse"] == b["rmse"] and np.array_equal(a["errors"], b["errors"])
    r0, r1 = metrics.rpe(est, gt), metrics.rpe(est, gt, valid=np.ones(n, bool))
    assert r0["trans_rmse"] == r1["trans_rmse"] and r0["rot_rmse_deg"] == r1["rot_rmse_deg"]
    # frames 3 and 7 have no GT pose (inf, as ScanNet writes it), frame 9 is flagged out by the caller
    gi = gt.copy()
    gi[3] = np.inf
    gi[7, 0, 0] = -np.inf
    valid = np.ones(n, bool)
    valid[9] = False
    keep = np.array([i for i in range(n) if i not in (3, 7, 9)])
    for align in (True, False):
        got, ref = metrics.ate(est, gi, align=align, valid=valid), metrics.ate(est[keep], gt[keep], align=align)
        assert got["rmse"] == ref["rmse"] and got["max"] == ref["max"] and np.array_equal(got["errors"], ref["errors"])
    got = metrics.rpe(est, gi, valid=valid)
    pairs = [i for i in range(n - 1) if i in keep and i + 1 in keep]
    ref_t = [metrics.rpe(est[[i, i + 1]], gt[[i, i + 1]])["trans_errors"][0] for i in pairs]
    ref_r = [metrics.rpe(est[[i, i + 1]], gt[[i, i + 1]])["rot_errors_deg"][0] for i in pairs]
    assert np.array_equal(got["trans_errors"], ref_t) and np.array_equal(got["rot_errors_deg"], ref_r)
    assert got["trans_rmse"] == float(np.sqrt(np.mean(np.square(ref_t))))
    got2 = metrics.rpe(est, gi, delta=2, valid=valid)
    assert len(got2["trans_errors"]) == len([i for i in range(n - 2) if i in keep and i + 2 in keep])
    with pytest.raises(ValueError):
        metrics.ate(est, gt, valid=np.ones(n - 1, bool))
    with pytest.raises(ValueError):
        metrics.ate(est, np.full_like(gt, np.inf), valid=np.ones(n, bool))


def test_relabel_struct_matches_header():
    from vmap_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    body = src[src.index("typedef struct vmb_relabel_args"):src.index("} vmb_relabel_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"[\s\*]([a-z_0-9]+)\s*(?:\[\d+\])?\s*[;,]", body)
    assert names == [f[0] for f in _lib.RelabelArgs._fields_]
    assert "vmb_store_relabel" in _lib.EXPORTS and "int vmb_store_relabel(vmb_handle* h, const vmb_relabel_args* a" in src


def test_slam_refuses_association_where_it_does_not_apply():
    from vmap_b200.cfg import Config, replica_room0_dict
    from vmap_b200.slam import Slam
    marker = object()
    with pytest.raises(ValueError, match="iMAP"):
        Slam(Config(config_dict=replica_room0_dict(imap=True)), assoc=marker)
    with pytest.raises(ValueError, match="map=False"):
        Slam(Config(config_dict=replica_room0_dict()), map=False, groups=[], assoc=marker)
