"""Config: JSON -> flat attribute bag with the reference's attribute names (cfg.py:6-91),
so code written against ``cfg.Config`` (train.py, vmap.py, trainer.py) reads the same fields."""
from __future__ import annotations

import json
import os
import weakref

import numpy as np


def _load_matrix_txt(path):
    return np.loadtxt(path)


_POSE_LR: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


class Config:
    @property
    def pose_lr(self) -> float:
        """optimizer.args.pose_lr, the camera-tracking rate (vmap_b200/track.py).  Every shipped config carries it and
        the reference never reads it, so it is kept out of the instance's attribute bag, which stays the reference's."""
        return _POSE_LR.get(self, 0.001)

    # pose_lr travels with copies and pickles of the config, outside the attribute bag
    def __getstate__(self):
        return dict(self.__dict__, _pose_lr=self.pose_lr)

    def __setstate__(self, state):
        state = dict(state)
        _POSE_LR[self] = state.pop("_pose_lr", 0.001)
        self.__dict__.update(state)

    def __init__(self, config_file=None, config_dict=None):
        if config_dict is None:
            with open(config_file) as f:
                config_dict = json.load(f)
        c = config_dict
        tr, ds, rd, md, cam, vis = c["trainer"], c["dataset"], c["render"], c["model"], c["camera"], c["vis"]
        # training strategy (cfg.py:13-21)
        self.do_bg = bool(tr["do_bg"])
        self.training_device = tr["train_device"]
        self.data_device = tr["data_device"]
        self.max_n_models = tr["n_models"]
        self.live_mode = bool(ds["live"])
        self.keep_live_time = ds["keep_alive"]
        self.imap_mode = tr["imap_mode"]
        self.training_strategy = tr["training_strategy"]
        self.obj_id = -1
        # dataset (cfg.py:24-26)
        self.dataset_format = ds["format"]
        self.dataset_dir = ds["path"]
        self.depth_scale = 1 / tr["scale"]
        # camera (cfg.py:28-60)
        self.min_depth, self.max_depth = rd["depth_range"][0], rd["depth_range"][1]
        self.mh, self.mw = cam["mh"], cam["mw"]
        self.height, self.width = cam["h"], cam["w"]
        self.H = self.height - 2 * self.mh
        self.W = self.width - 2 * self.mw
        if "fx" in cam:
            self.fx, self.fy = cam["fx"], cam["fy"]
            self.cx, self.cy = cam["cx"] - self.mw, cam["cy"] - self.mh
        else:   # ScanNet keeps its intrinsics beside the data (cfg.py:41-46)
            k = _load_matrix_txt(os.path.join(self.dataset_dir, "intrinsic/intrinsic_depth.txt"))
            self.fx, self.fy = k[0, 0], k[1, 1]
            self.cx, self.cy = k[0, 2] - self.mw, k[1, 2] - self.mh
        if "distortion" in cam:
            self.distortion_array = np.array(cam["distortion"])
        elif "k1" in cam:
            self.distortion_array = np.array([cam[k] for k in ("k1", "k2", "p1", "p2", "k3", "k4", "k5", "k6")])
        else:
            self.distortion_array = None
        # training (cfg.py:63-82)
        self.win_size = md["window_size"]
        self.n_iter_per_frame = rd["iters_per_frame"]
        self.n_per_optim = rd["n_per_optim"]
        self.n_samples_per_frame = self.n_per_optim // self.win_size
        self.win_size_bg = md["window_size_bg"]
        self.n_per_optim_bg = rd["n_per_optim_bg"]
        self.n_samples_per_frame_bg = self.n_per_optim_bg // self.win_size_bg
        self.keyframe_buffer_size = md["keyframe_buffer_size"]
        self.keyframe_step = md["keyframe_step"]
        self.keyframe_step_bg = md["keyframe_step_bg"]
        self.obj_scale = md["obj_scale"]
        self.bg_scale = md["bg_scale"]
        self.hidden_feature_size = md["hidden_feature_size"]
        self.hidden_feature_size_bg = md["hidden_feature_size_bg"]
        self.n_bins_cam2surface = rd["n_bins_cam2surface"]
        self.n_bins_cam2surface_bg = rd["n_bins_cam2surface_bg"]
        self.n_bins = rd["n_bins"]
        self.n_unidir_funcs = md["n_unidir_funcs"]
        self.surface_eps = md["surface_eps"]
        self.stop_eps = md["other_eps"]
        # optimiser (cfg.py:85-86)
        self.learning_rate = c["optimizer"]["args"]["lr"]
        self.weight_decay = c["optimizer"]["args"]["weight_decay"]
        _POSE_LR[self] = float(c["optimizer"]["args"].get("pose_lr", 0.001))
        # vis (cfg.py:89-92)
        self.vis_device = vis["vis_device"]
        self.n_vis_iter = vis["n_vis_iter"]
        self.live_voxel_size = vis["live_voxel_size"]
        self.grid_dim = vis["grid_dim"]


def replica_room0_dict(imap: bool = False, device: str = "cuda:0") -> dict:
    """The shipped Replica room0 settings (configs/Replica/config_replica_room0_{vMAP,iMAP}.json)
    as a dict, for synthetic runs where the dataset path is irrelevant."""
    d = {
        "dataset": {"live": 0, "path": "", "format": "Replica", "keep_alive": 20},
        "optimizer": {"args": {"lr": 0.001, "weight_decay": 0.013, "pose_lr": 0.001}},
        "trainer": {"imap_mode": 0, "do_bg": 1, "n_models": 100, "train_device": device, "data_device": device,
                    "training_strategy": "vmap", "epochs": 1000000, "scale": 1000.0},
        "render": {"depth_range": [0.0, 8.0], "n_bins": 9, "n_bins_cam2surface": 1, "n_bins_cam2surface_bg": 5,
                   "iters_per_frame": 20, "n_per_optim": 120, "n_per_optim_bg": 1200},
        "model": {"n_unidir_funcs": 5, "obj_scale": 2.0, "bg_scale": 5.0, "color_scaling": 5.0,
                  "opacity_scaling": 10.0, "gt_scene": 1, "surface_eps": 0.1, "other_eps": 0.05,
                  "keyframe_buffer_size": 20, "keyframe_step": 25, "keyframe_step_bg": 50, "window_size": 5,
                  "window_size_bg": 10, "hidden_layers_block": 1, "hidden_feature_size": 32,
                  "hidden_feature_size_bg": 128},
        "camera": {"w": 1200, "h": 680, "fx": 600.0, "fy": 600.0, "cx": 599.5, "cy": 339.5, "mw": 0, "mh": 0},
        "vis": {"vis_device": device, "n_vis_iter": 500, "n_bins_fine_vis": 10, "im_vis_reduce": 10,
                "grid_dim": 256, "live_vis": 1, "live_voxel_size": 0.005},
    }
    if imap:
        d["trainer"].update(imap_mode=1, do_bg=0, n_models=1)
        d["render"].update(n_bins_cam2surface=5, n_per_optim=4800)
        d["model"].update(obj_scale=5.0, keyframe_step=50, hidden_feature_size=256)
    return d
