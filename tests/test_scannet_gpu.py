"""GPU tests of ScanNet association (vmb_assoc_*, vmap_b200/scannet.py): bitwise labels / bbox_dict against the
reference goldens and the restated oracle, track counts, boxes, edge frames and a drop-in loader run."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import scannet_oracle as so

pytestmark = pytest.mark.gpu


def _cfg(root, imap=False):
    from vmap_b200.cfg import Config
    d = {
        "dataset": {"live": 0, "path": root, "format": "ScanNet", "keep_alive": 20},
        "optimizer": {"args": {"lr": 0.001, "weight_decay": 0.013, "pose_lr": 0.001}},
        "trainer": {"imap_mode": int(imap), "do_bg": 1, "n_models": 100, "train_device": "cuda:0",
                    "data_device": "cuda:0", "training_strategy": "vmap", "epochs": 1000000, "scale": 1000.0},
        "render": {"depth_range": [0.0, 6.0], "n_bins": 9, "n_bins_cam2surface": 1, "n_bins_cam2surface_bg": 5,
                   "iters_per_frame": 20, "n_per_optim": 120, "n_per_optim_bg": 1200},
        "model": {"n_unidir_funcs": 5, "obj_scale": 3.0, "bg_scale": 10.0, "color_scaling": 5.0,
                  "opacity_scaling": 10.0, "gt_scene": 1, "surface_eps": 0.1, "other_eps": 0.05,
                  "keyframe_buffer_size": 20, "keyframe_step": 25, "keyframe_step_bg": 50, "window_size": 5,
                  "window_size_bg": 10, "hidden_layers_block": 1, "hidden_feature_size": 32,
                  "hidden_feature_size_bg": 128},
        "camera": {"w": 640, "h": 480, "mw": 10, "mh": 10},
        "vis": {"vis_device": "cuda:0", "n_vis_iter": 10000000, "n_bins_fine_vis": 10, "im_vis_reduce": 10,
                "grid_dim": 256, "live_vis": 1, "live_voxel_size": 0.005},
    }
    return Config(config_dict=d)


def gpu_run(root, n_trackers):
    from vmap_b200 import scannet
    cfg = _cfg(root)
    ds = scannet.ScanNet(cfg, n_trackers=n_trackers)
    out = []
    for i, smp in enumerate(scannet._Loader(ds, n_trackers)):
        tr = ds.trackers[i % n_trackers]
        snap = {k: (d.bbox3D.center, d.bbox3D.R, d.bbox3D.extent, len(d.pc), d.cmp_cnt)
                for k, d in tr.inst_dict.items()}
        smp = dict(smp, obj=smp["obj"].cpu().numpy(), bbox_dict={k: v.numpy() for k, v in smp["bbox_dict"].items()})
        out.append((smp, snap))
    return out


def assert_same(results, ref):
    assert len(results) == len(ref)
    for i, ((s, t), (rs, rt)) in enumerate(zip(results, ref)):
        np.testing.assert_array_equal(s["obj"], np.asarray(rs["obj"]), err_msg=f"frame {i} labels")
        assert sorted(s["bbox_dict"]) == sorted(rs["bbox_dict"]), i
        for k in rs["bbox_dict"]:
            np.testing.assert_array_equal(s["bbox_dict"][k], np.asarray(rs["bbox_dict"][k]).reshape(4))
        assert sorted(t) == sorted(rt), i
        for k in rt:
            assert t[k][3] == rt[k][3] and t[k][4] == rt[k][4], (i, k)
            np.testing.assert_allclose(t[k][0], rt[k][0], rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(t[k][2], rt[k][2], rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(np.abs(np.sum(t[k][1] * rt[k][1], axis=0)), 1.0, atol=1e-9)


def golden_as_results(g):
    out = []
    for i in range(int(g["n_frames"])):
        keys = list(g[f"bbox_keys_{i}"])
        smp = {"obj": g[f"obj_{i}"].astype(np.int64), "bbox_dict": dict(zip(keys, g[f"bbox_{i}"]))}
        ids = list(g[f"track_ids_{i}"])
        tracks = {k: (g[f"track_center_{i}"][j], g[f"track_R_{i}"][j], g[f"track_extent_{i}"][j],
                      int(g[f"track_npts_{i}"][j]), int(g[f"track_cmp_{i}"][j])) for j, k in enumerate(ids)}
        out.append((smp, tracks))
    return out


@pytest.mark.parametrize("name,n_trackers", [("seq", 1), ("workers", 4)])
def test_gpu_equals_reference_golden(golden_dir, name, n_trackers):
    g = np.load(os.path.join(golden_dir, f"ref_scannet_{name}.npz"))
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=int(g["seed"]), n_frames=int(g["n_frames"]))
        res = gpu_run(root, n_trackers)
    assert_same(res, golden_as_results(g))


@pytest.mark.parametrize("seed,n_extra,id_base", [(5, 12, 10), (7, 20, 1030)])
def test_gpu_equals_oracle_on_extra_sequences(seed, n_extra, id_base):
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=seed, n_frames=8, n_extra=n_extra, id_base=id_base, inf_frame=-1)
        ref = so.run(root, n_trackers=1)
        res = gpu_run(root, 1)
    assert_same(res, ref)
    assert any(k >= 1024 for k in res[-1][1]) == (id_base >= 1024)


def test_empty_and_background_frames_and_imap():
    from vmap_b200.scannet import InstanceTracker, ScanNet
    tr = InstanceTracker(500.0, 500.0, 100.0, 80.0, "cuda:0")
    W, H = 200, 160
    depth = torch.full((W, H), 2.0, device="cuda")
    for inst, sem in ((torch.zeros((W, H), dtype=torch.int32), None),                      # empty frame
                      (torch.full((W, H), 3, dtype=torch.int32), torch.full((W, H), 1, dtype=torch.int32))):  # wall
        lab, bb = tr.frame(inst, depth, T=np.eye(4), sem=sem)
        assert torch.all(lab == 0) and list(bb) == [0]
        assert bb[0].tolist() == [0, W, 0, H]
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=1, n_frames=3)
        smp = ScanNet(_cfg(root, imap=True))[0]
        assert torch.all(smp["obj"] == 0) and list(smp["bbox_dict"]) == [0]


def test_box_filter_mirror_equals_oracle():
    from vmap_b200 import utils
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=3, n_frames=3)
        seq = so.Sequence(root)
        inst_dict, tracks = {}, {}
        fx, fy, cx, cy = seq.intr
        intr = so.o3d.PinholeCameraIntrinsic(620, 460, fx, fy, cx, cy)
        for i in range(3):
            color, depth, T, inst, sem = so.load_frame(root, i, 620, 460, 10, 1 / 1000.0, 6.0, seq.poses)
            masks, classes = [], []
            for k in np.unique(inst):
                m = inst == k
                if int(sem[m].min()) in so.BG_CLASSES:
                    continue
                masks.append(m)
                classes.append(int(k))
            T_CW = np.linalg.inv(T)
            got = utils.box_filter(masks, classes, depth, inst_dict, intr, T_CW, min_pixels=1500)
            ref = so.box_filter(inst, sem, depth, tracks, seq.intr, np.linalg.inv(T_CW))
            assert got.dtype == np.int64 and got.shape == depth.shape
            np.testing.assert_array_equal(got, ref)
            assert sorted(inst_dict) == sorted(tracks)


def test_dropin_append_loop_creates_oracle_ids():
    """train.py:105-164's append loop on init_loader(cfg): the objects created are the oracle's ids."""
    from vmap_b200 import scannet
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=3, n_frames=6)
        cfg = _cfg(root)
        loader = scannet.init_loader(cfg)
        it = iter(loader)
        vis_dict = {}
        for frame_id in range(len(loader)):
            sample = next(it)
            rgb = sample["image"].to(cfg.data_device)
            depth = sample["depth"].to(cfg.data_device)
            twc = sample["T"].to(cfg.data_device)
            bbox_dict = sample["bbox_dict"]
            inst = sample["obj"].to(cfg.data_device)
            assert rgb.dtype == torch.uint8 and rgb.shape == (620, 460, 3)
            assert depth.dtype == torch.float32 and twc.dtype == torch.float64 and inst.dtype == torch.int64
            for obj_id in torch.unique(inst):
                if obj_id == -1:
                    continue
                obj_id = int(obj_id)
                state = torch.zeros_like(inst, dtype=torch.uint8, device=cfg.data_device)
                state[inst == obj_id] = 1
                state[inst == -1] = 2
                bbox = bbox_dict[obj_id]
                vis_dict.setdefault(obj_id, []).append((frame_id, int(state.sum()), bbox.tolist()))
        ref = so.run(root, n_trackers=4)
    ref_ids = set()
    for smp, _ in ref:
        ref_ids |= set(np.unique(smp["obj"]).tolist()) - {-1}
    assert set(vis_dict) == ref_ids
