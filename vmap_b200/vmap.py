"""sceneObject / cameraInfo / performance_measure with the reference's call surface
(vmap.py:17-29, 90-491, 494-524).  The keyframe buffers are the reference's tensors
(same shapes / dtypes, images stored [W, H]); the arithmetic of
``get_training_samples`` (vmap.py:319-459) runs in the batched CUDA sampler (K3):
``sample_all`` draws for every object of the frame in ONE launch (replacing the Python
loop of train.py:208-218 and the stack + /255 of train.py:255-260), and the per-object
method is the same kernel with one object.
"""
from __future__ import annotations

import copy
import os
import random
from time import perf_counter_ns
from typing import Dict, List, Optional

import numpy as np
import torch

from . import trainer as trainer_mod
from .sampler import BatchedSampler, KeyframeSet, KeyframeTables, _latest2


class performance_measure:
    """Wall-clock context manager that prints ms (vmap.py:17-29); kept as the reference's
    only timing hook.  Pass ``sync=True`` to bracket with cuda synchronize."""

    def __init__(self, name, sync: bool = False) -> None:
        self.name, self.sync = name, sync

    def __enter__(self):
        if self.sync and torch.cuda.is_available():
            torch.cuda.synchronize()
        self.start_time = perf_counter_ns()

    def __exit__(self, type, value, tb):
        if self.sync and torch.cuda.is_available():
            torch.cuda.synchronize()
        self.end_time = perf_counter_ns()
        self.exec_time = self.end_time - self.start_time
        print(f"{self.name} excution time: {(self.exec_time)/1000000:.2f} ms")


class cameraInfo:
    """Ray-direction cache [W,H,3] = ((u-cx)/fx, (v-cy)/fy, 1) (vmap.py:494-524)."""

    def __init__(self, cfg) -> None:
        self.device = cfg.data_device
        self.width, self.height = cfg.W, cfg.H
        self.fx, self.fy, self.cx, self.cy = cfg.fx, cfg.fy, cfg.cx, cfg.cy
        self.rays_dir_cache = self.get_rays_dirs()

    def get_rays_dirs(self, depth_type="z"):
        if depth_type != "z":
            raise Exception("Get camera rays directions with euclidean depth not yet implemented")
        u = (torch.arange(self.width, device=self.device) - self.cx) / self.fx
        v = (torch.arange(self.height, device=self.device) - self.cy) / self.fy
        dirs = torch.ones((self.width, self.height, 3), device=self.device)
        dirs[:, :, 0] = u[:, None]
        dirs[:, :, 1] = v
        return dirs


_SAMPLERS: Dict[tuple, BatchedSampler] = {}
_CALLS = [0]


def _sampler_for(obj) -> BatchedSampler:
    key = (str(obj.data_device), obj.n_bins_cam2surface, obj.n_bins, obj.surface_eps, obj.stop_eps, obj.min_bound)
    if key not in _SAMPLERS:
        _SAMPLERS[key] = BatchedSampler(obj.data_device, obj.n_bins_cam2surface, obj.n_bins, obj.surface_eps,
                                        obj.stop_eps, obj.min_bound)
    return _SAMPLERS[key]


def sample_all(objects: List["sceneObject"], n_frames: int, n_samples: int, cached_rays_dir: torch.Tensor,
               seed: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """One launch for every object: stacked {pcs [B,N,S,3], z [B,N,S], gt_depth [B,N],
    gt_colour [B,N,3] (already /255), sem [B,N] u8, mask_depth [B,N] bool}, N = n_frames*n_samples.
    All objects must share the sampling configuration (objects vs. the background model differ)."""
    smp = _sampler_for(objects[0])
    _CALLS[0] += 1
    if seed is None:
        seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
    store = objects[0].store
    if store is not None:                                  # shared keyframe store: (slot, bbox) tables only
        assert all(o.store is store for o in objects), "objects of one launch must share the FrameStore"
        return smp.sample_store(store, keyframe_tables(objects), n_frames, n_samples, cached_rays_dir,
                                seed=seed, offset=_CALLS[0])
    return smp.sample([o.keyframe_set() for o in objects], n_frames, n_samples, cached_rays_dir,
                      seed=seed, offset=_CALLS[0])


def keyframe_tables(objects: List["sceneObject"]) -> KeyframeTables:
    """Pack the (store slot, bbox) tables of shared-store objects for one sampler launch."""
    return KeyframeTables(torch.tensor([o.kf_store_slot for o in objects], dtype=torch.int32),
                          torch.stack([o.bbox for o in objects]),
                          [int(o.obj_id) for o in objects], [o.n_keyframes for o in objects],
                          [_latest2(o.lastest_kf_queue[-2:] if len(o.lastest_kf_queue) >= 2 else [0, 0])
                           for o in objects])


class sceneObject:
    """Per-object keyframe buffers + sampler entry point (vmap.py:90-491)."""

    def __init__(self, cfg, obj_id, rgb: Optional[torch.Tensor], depth: Optional[torch.Tensor],
                 mask: Optional[torch.Tensor], bbox_2d: torch.Tensor, t_wc: torch.Tensor, live_frame_id,
                 store=None, frame_slot: Optional[int] = None) -> None:
        """``store`` / ``frame_slot``: shared keyframe store mode (keyframes.FrameStore) -- the frame already
        lives in ``store`` slot ``frame_slot``; rgb / depth / mask are not copied (pass None) and the object
        keeps only (slot, bbox) per keyframe.  Without ``store`` this is the reference's per-object layout."""
        self.do_bg = cfg.do_bg
        self.obj_id = obj_id
        self.data_device = cfg.data_device
        self.training_device = cfg.training_device
        self.store = store
        if store is None:
            assert rgb.shape[:2] == depth.shape and rgb.shape[:2] == mask.shape
        else:
            assert frame_slot is not None
        assert bbox_2d.shape == (4,) and t_wc.shape == (4, 4)
        bg = self.do_bg and self.obj_id == 0                     # vmap.py:109-118
        self.obj_scale = cfg.bg_scale if bg else cfg.obj_scale
        self.hidden_feature_size = cfg.hidden_feature_size_bg if bg else cfg.hidden_feature_size
        self.n_bins_cam2surface = cfg.n_bins_cam2surface_bg if bg else cfg.n_bins_cam2surface
        self.keyframe_step = cfg.keyframe_step_bg if bg else cfg.keyframe_step
        self.frames_width, self.frames_height = (store.W, store.H) if store is not None else (rgb.shape[0], rgb.shape[1])
        self.min_bound, self.max_bound = cfg.min_depth, cfg.max_depth
        self.n_bins, self.n_unidir_funcs = cfg.n_bins, cfg.n_unidir_funcs
        self.surface_eps, self.stop_eps = cfg.surface_eps, cfg.stop_eps
        self.n_keyframes = 1
        self.kf_pointer = None
        self.keyframe_buffer_size = cfg.keyframe_buffer_size
        self.kf_id_dict = {live_frame_id: 0}                     # frame id -> buffer slot
        self.kf_buffer_full = False
        self.frame_cnt = 0
        self.lastest_kf_queue = []
        KF, W, H, dev = self.keyframe_buffer_size, self.frames_width, self.frames_height, self.data_device
        self.rgb_idx, self.state_idx = slice(0, 3), slice(3, 4)
        self.other_obj, self.this_obj, self.unknown_obj = 0, 1, 2
        if store is None:
            self.bbox = torch.empty(KF, 4, device=dev)           # [u low, u high, v low, v high]
            self.rgbs_batch = torch.empty(KF, W, H, 4, dtype=torch.uint8, device=dev)
            self.depth_batch = torch.empty(KF, W, H, dtype=torch.float32, device=dev)
            self.t_wc_batch = torch.empty(KF, 4, 4, dtype=torch.float32, device=dev)
        else:                                                    # host tables only: KF x (slot, bbox)
            self.bbox = torch.zeros(KF, 4)
            self.kf_store_slot = [0] * KF                        # unused entries point at slot 0 (never sampled)
            self._held = [False] * KF
            self.rgbs_batch = self.depth_batch = self.t_wc_batch = None
        self._store(0, rgb, depth, mask, bbox_2d, t_wc, frame_slot)
        tcfg = copy.deepcopy(cfg)
        tcfg.obj_id, tcfg.hidden_feature_size, tcfg.obj_scale = self.obj_id, self.hidden_feature_size, self.obj_scale
        self.trainer = trainer_mod.Trainer(tcfg)
        self.bbox3d = None
        self.pc = []
        self.obj_center = torch.tensor(0.0)

    def _store(self, slot, rgb, depth, mask, bbox_2d, t_wc, frame_slot=None):
        if self.store is not None:
            assert frame_slot is not None, "shared-store object: pass frame_slot"
            self.store.acquire(frame_slot)
            if self._held[slot]:
                self.store.release(self.kf_store_slot[slot])
            self.kf_store_slot[slot], self._held[slot] = int(frame_slot), True
            self.bbox[slot] = torch.as_tensor(bbox_2d, dtype=torch.float32).cpu()
            return
        self.rgbs_batch[slot, :, :, self.rgb_idx] = rgb
        self.rgbs_batch[slot, :, :, self.state_idx] = mask[..., None]
        self.depth_batch[slot] = depth
        self.t_wc_batch[slot] = t_wc
        self.bbox[slot] = bbox_2d

    def _slot_to_frame(self, slot, frame_id):
        for k in [k for k, v in self.kf_id_dict.items() if v == slot]:
            del self.kf_id_dict[k]
        self.kf_id_dict[frame_id] = slot

    def release_frames(self):
        """Shared-store mode: give the object's frame references back (object deleted)."""
        if self.store is not None:
            for k, held in enumerate(self._held):
                if held:
                    self.store.release(self.kf_store_slot[k])
                    self._held[k] = False

    def append_keyframe(self, rgb, depth, mask, bbox_2d, t_wc, frame_id=1, frame_slot=None):
        """vmap.py:208-263: a new keyframe every ``keyframe_step`` frames, otherwise the newest
        slot is overwritten; once the buffer is full a random old keyframe is recycled.
        Shared-store mode: pass ``frame_slot`` (rgb / depth / mask may be None)."""
        assert bbox_2d.shape == (4,) and t_wc.shape == (4, 4)
        assert self.n_keyframes <= self.keyframe_buffer_size - 1
        if self.store is None:
            assert rgb.shape[:2] == depth.shape and rgb.shape[:2] == mask.shape
            assert rgb.dtype == torch.uint8 and mask.dtype == torch.uint8 and depth.dtype == torch.float32
        is_kf = (self.frame_cnt % self.keyframe_step == 0) or self.n_keyframes == 1
        if self.n_keyframes == self.keyframe_buffer_size - 1:
            self.kf_buffer_full = True
            if self.kf_pointer is None:
                self.kf_pointer = self.n_keyframes
            self._store(self.kf_pointer, rgb, depth, mask, bbox_2d, t_wc, frame_slot)
            self._slot_to_frame(self.kf_pointer, frame_id)
            if is_kf:
                self.lastest_kf_queue.append(self.kf_pointer)
                _, self.kf_pointer = self.prune_keyframe()
                print("pruned kf id ", self.kf_pointer)
        elif not is_kf:
            self._store(self.n_keyframes - 1, rgb, depth, mask, bbox_2d, t_wc, frame_slot)
            self._slot_to_frame(self.n_keyframes - 1, frame_id)
        else:
            self.kf_id_dict[frame_id] = self.n_keyframes
            self._store(self.n_keyframes, rgb, depth, mask, bbox_2d, t_wc, frame_slot)
            self.lastest_kf_queue.append(self.n_keyframes)
            self.n_keyframes += 1
        self.frame_cnt += 1
        if len(self.lastest_kf_queue) > 2:
            self.lastest_kf_queue = self.lastest_kf_queue[-2:]

    def prune_keyframe(self):
        return random.choice(list(self.kf_id_dict.items())[:-2])    # never the latest two (vmap.py:265-268)

    def keyframe_set(self) -> KeyframeSet:
        latest = self.lastest_kf_queue[-2:] if len(self.lastest_kf_queue) >= 2 else [0, 0]
        return KeyframeSet(self.rgbs_batch, self.depth_batch, self.t_wc_batch, self.bbox, self.n_keyframes, latest)

    def get_training_samples(self, n_frames, n_samples, cached_rays_dir):
        """The reference's 6-tuple (vmap.py:459): rgb [F,P,3] u8, depth [F,P], valid_depth_mask
        [F*P] bool, obj_labels [F*P] u8, pcs [F,P,S,3], z [F,P,S]."""
        smp = _sampler_for(self)
        _CALLS[0] += 1
        seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
        if self.store is not None:
            o = smp.sample_store(self.store, keyframe_tables([self]), n_frames, n_samples, cached_rays_dir,
                                 seed=seed, offset=_CALLS[0], want_u8=True)
        else:
            o = smp.sample([self.keyframe_set()], n_frames, n_samples, cached_rays_dir,
                           seed=seed, offset=_CALLS[0], want_u8=True)
        S = o["z"].shape[-1]
        return (o["gt_rgb_u8"][0].view(n_frames, n_samples, 3), o["gt_depth"][0].view(n_frames, n_samples),
                o["mask_depth"][0], o["sem"][0], o["pcs"][0].view(n_frames, n_samples, S, 3),
                o["z"][0].view(n_frames, n_samples, S))

    def get_bound(self, intrinsic_open3d):
        """Oriented 3-D bound of the object (vmap.py:270-315).  The object's pixels of its first ``n_keyframes``
        keyframes with depth > 0 are unprojected on the GPU (K5); their exact convex hull and its minimum-volume box
        are computed there too (K8, mesh.oriented_bounds_gpu), extents clamped to >= 0.10.  Stores a picklable utils.BoundingBox in
        ``self.bbox3d`` (it goes into checkpoints) and returns an open3d OrientedBoundingBox when open3d is installed
        (train.py:367 adds it to the viewer), the BoundingBox otherwise; None when the points are too few or flat.
        ``intrinsic_open3d``: an open3d PinholeCameraIntrinsic or a 3x3 matrix."""
        from . import mesh, utils
        pts = mesh.unproject_object(self, mesh.intrinsic_matrix(intrinsic_open3d))
        try:
            center, R, extents = mesh.oriented_bounds_gpu(pts)
        except ValueError:
            print("too few pcs obj ")
            return None
        extents = np.maximum(extents, 0.10)                  # at least rendering 10cm (vmap.py:298-299, 306-307)
        bbox = utils.BoundingBox()
        bbox.center, bbox.R, bbox.extent = center, R, extents
        self.bbox3d = bbox
        print("obj ", self.obj_id)
        print("bound ", f"center {center}, extent {extents}")
        print("kf id dict ", self.kf_id_dict)
        try:
            import open3d
        except ImportError:
            return bbox
        bbox3d = open3d.geometry.OrientedBoundingBox(center, R, extents)
        bbox3d.color = (255, 0, 0)
        return bbox3d

    def save_checkpoints(self, path, epoch):
        """Same file layout and keys as vmap.py:461-476."""
        f = os.path.join(path, "obj_" + str(self.obj_id) + "_frame_" + str(epoch) + ".pth")
        torch.save({"epoch": epoch,
                    "FC_state_dict": {k: v.detach().clone() for k, v in self.trainer.fc_occ_map.state_dict().items()},
                    "PE_state_dict": {k: v.detach().clone() for k, v in self.trainer.pe.state_dict().items()},
                    "obj_id": self.obj_id, "bbox": self.bbox3d, "obj_scale": self.trainer.obj_scale}, f)

    def load_checkpoints(self, ckpt_file):
        """vmap.py:478-491; parameters bound to a packed ensemble are written in place."""
        if not os.path.exists(ckpt_file):
            print("ckpt not exist ", ckpt_file)
            return
        ck = torch.load(ckpt_file, weights_only=False)
        with torch.no_grad():
            for k, p in self.trainer.fc_occ_map.named_parameters():
                p.copy_(ck["FC_state_dict"][k].to(p.device))
            self.trainer.pe.B_layer.weight.copy_(ck["PE_state_dict"]["B_layer.weight"].to(self.trainer.pe.B_layer.weight.device))
        self.obj_id, self.bbox3d = ck["obj_id"], ck["bbox"]
        self.trainer.obj_scale = ck["obj_scale"]
        pe = self.trainer.pe
        if "scale" in ck["PE_state_dict"]:          # persistent buffer of UniDirsEmbed (embedding.py:80): load_state_dict restores it
            with torch.no_grad():
                pe.scale.copy_(ck["PE_state_dict"]["scale"].to(pe.scale.device))
        b = getattr(self.trainer.fc_occ_map, "_vmb_binding", None)
        if b is not None and b[0]() is not None:
            ens, row = b[0](), b[1]
            ens.scale[row] = float(pe.scale)         # the kernels read the packed copy
            ens.reset_optimizer_row(row)             # freshly loaded weights start AdamW from scratch, like a new param group
            ens.refresh_image()
