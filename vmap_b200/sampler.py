"""Batched depth-guided ray sampler (K3) -- host side.

Replaces the per-object Python loop of train.py:208-218 over
``sceneObject.get_training_samples`` (vmap.py:319-459) and the stack + /255 of
train.py:255-260 with one kernel launch for all objects of the frame.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import torch

from . import _lib


@dataclass
class KeyframeSet:
    """The per-object buffers the sampler reads (sceneObject fields, vmap.py:137-176)."""
    rgbs_batch: torch.Tensor      # [KF,W,H,4] u8 (rgb + state)
    depth_batch: torch.Tensor     # [KF,W,H] f32
    t_wc_batch: torch.Tensor      # [KF,4,4] f32
    bbox: torch.Tensor            # [KF,4] f32
    n_keyframes: int
    latest_kf: Sequence[int]      # lastest_kf_queue[-2:]


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class BatchedSampler:
    def __init__(self, device="cuda:0", n_bins_cam2surface=1, n_bins=9, surface_eps=0.1, stop_eps=0.05,
                 min_bound=0.0, max_obj=1024):
        self.lib = _lib.lib()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.VmbError("BatchedSampler needs a CUDA device: there is no CPU fallback")
        self.n1, self.n2 = n_bins_cam2surface, n_bins
        self.eps, self.oeps, self.min_bound = surface_eps, stop_eps, min_bound
        self._handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(None, self.lib.vmb_create(C.byref(self._handle), self.device.index or 0, max_obj, 32, 6),
                       "vmb_create")
        lim = torch.zeros(3, 33)
        for row, n in enumerate((self.n1 + self.n2, self.n1, self.n2)):
            lim[row, :n + 1] = torch.linspace(0, 1, n + 1, dtype=torch.float32)     # vmap.py:48
        self.bin_limits = lim.to(self.device)
        self._keep = None

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self.lib.vmb_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def _outputs(self, B, N, S, want_u8):
        dev = self.device
        out = {
            "pcs": torch.empty(B, N, S, 3, dtype=torch.float32, device=dev),
            "z": torch.empty(B, N, S, dtype=torch.float32, device=dev),
            "gt_depth": torch.empty(B, N, dtype=torch.float32, device=dev),
            "gt_colour": torch.empty(B, N, 3, dtype=torch.float32, device=dev),
            "sem": torch.empty(B, N, dtype=torch.uint8, device=dev),
            "mask_depth": torch.empty(B, N, dtype=torch.bool, device=dev),
        }
        if want_u8:
            out["gt_rgb_u8"] = torch.empty(B, N, 3, dtype=torch.uint8, device=dev)
        return out

    def _launch(self, a, out, B, n_frames, n_pix, W, H, rays_dir, seed, offset, inject, keep, offset_dev=None,
                camera_frame=False, kf_out=None):
        dev = self.device
        if kf_out is not None:
            assert kf_out.dtype == torch.int32 and kf_out.shape == (B, n_frames) and kf_out.is_contiguous()
        a.camera_frame, a.kf_out = int(bool(camera_frame)), _p(kf_out)
        a.n_obj, a.n_frames, a.n_pix = B, n_frames, n_pix
        a.n_bins_cam2surface, a.n_bins, a.width, a.height = self.n1, self.n2, W, H
        a.min_bound, a.surface_eps, a.stop_eps = self.min_bound, self.eps, self.oeps
        a.rays_dir, a.bin_limits = _p(rays_dir), _p(self.bin_limits)
        a.seed, a.offset = seed, offset
        a.offset_dev = _p(offset_dev)
        inj = None
        if inject is not None:
            inj = {k: v.to(dev).contiguous() for k, v in inject.items()}
            a.inj_kf, a.inj_u_w, a.inj_u_h = _p(inj["kf"]), _p(inj["u_w"]), _p(inj["u_h"])
            a.inj_u_z, a.inj_nrm = _p(inj["u_z"]), _p(inj["nrm"])
        a.pcs, a.z_vals, a.gt_depth, a.gt_colour = _p(out["pcs"]), _p(out["z"]), _p(out["gt_depth"]), _p(out["gt_colour"])
        a.gt_rgb_u8 = _p(out.get("gt_rgb_u8"))
        a.sem, a.mask_depth = _p(out["sem"]), _p(out["mask_depth"])
        with torch.cuda.device(dev):
            _lib.check(self._handle, self.lib.vmb_sample(
                self._handle, C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "vmb_sample")
        self._keep = (inj, keep)      # alive until the next call (async launch)
        return out

    def sample(self, objects: List[KeyframeSet], n_frames: int, n_pix: int, rays_dir: torch.Tensor,
               seed: int = 0, offset: int = 0, inject: Optional[Dict[str, torch.Tensor]] = None,
               want_u8: bool = False, tables: Optional["SamplerTables"] = None, out=None, offset_dev=None,
               camera_frame: bool = False, kf_out: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """Per-object keyframe buffers (the reference's layout, vmap.py:137-176).
        ``tables`` / ``out`` / ``offset_dev``: persistent table + output buffers and a device draw counter, for
        CUDA-graph capture of a whole frame (frame.FrameLoop); with ``tables`` the caller has already filled and
        uploaded them and ``objects`` is ignored.  ``camera_frame``: take every keyframe pose as identity (camera-frame
        points); ``kf_out`` [B, n_frames] int32: receives the keyframe index of each draw."""
        dev = self.device
        N, S = n_frames * n_pix, self.n1 + self.n2
        if tables is None:
            tables = SamplerTables(dev, len(objects))
            tables.fill_objects(objects)
            tables.upload()
        B, (W, H) = tables.n_obj, tables.image_wh           # the tables, not ``objects``, define the launch
        out = out if out is not None else self._outputs(B, N, S, want_u8)
        assert out["pcs"].shape == (B, N, S, 3) and out["sem"].shape == (B, N)
        a = _lib.SampleArgs()
        tables.bind(a)
        return self._launch(a, out, B, n_frames, n_pix, W, H, rays_dir, seed, offset, inject, tables, offset_dev,
                            camera_frame, kf_out)

    def sample_store(self, store, tables, n_frames: int, n_pix: int, rays_dir: torch.Tensor,
                     seed: int = 0, offset: int = 0, inject: Optional[Dict[str, torch.Tensor]] = None,
                     want_u8: bool = False, out=None, offset_dev=None, camera_frame: bool = False,
                     kf_out: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """Shared keyframe store (keyframes.FrameStore): frames stored once, per-object (slot, bbox) tables,
        pixel state derived from the instance image.  Same draws / outputs as ``sample`` on per-object copies.
        ``tables``: a ``KeyframeTables`` (packed and uploaded here) or an already uploaded ``SamplerTables``.
        ``camera_frame`` / ``kf_out``: as ``sample``."""
        dev = self.device
        assert store.device == dev
        if isinstance(tables, KeyframeTables):
            kt = tables
            tables = SamplerTables(dev, kt.kf_slot.shape[0], kf_stride=kt.kf_slot.shape[1])
            tables.fill_store(kt)
            tables.upload()
        B = tables.n_obj
        N, S = n_frames * n_pix, self.n1 + self.n2
        out = out if out is not None else self._outputs(B, N, S, want_u8)
        assert out["pcs"].shape == (B, N, S, 3) and out["sem"].shape == (B, N)
        a = _lib.SampleArgs()
        a.store_rgbx, a.store_depth, a.store_inst, a.store_t_wc = _p(store.rgbx), _p(store.depth), _p(store.inst), _p(store.t_wc)
        tables.bind(a)
        return self._launch(a, out, B, n_frames, n_pix, store.W, store.H, rays_dir, seed, offset, inject, tables, offset_dev,
                            camera_frame, kf_out)


class SamplerTables:
    """The per-object tables of one sampler launch in ONE pinned host buffer with a device twin, so a frame needs a
    single small host->device copy -- and, being persistent, that copy and the launch can sit inside a captured
    CUDA graph (fill on the host, then ``upload``).

    per-object mode (int64 words): [4][B] pointers rgbs|depths|t_wc|bbox, then int32 pairs n_kf[B] | latest[B][2]
    store mode      (int32 words): kf_slot[B][KF] | bbox[B][KF][4] (f32 bits) | obj_id[B] | n_kf[B] | latest[B][2]"""

    def __init__(self, device, n_obj: int, kf_stride: int = 0):
        self.device, self.n_obj, self.kf_stride = torch.device(device), n_obj, kf_stride
        B, KF = n_obj, kf_stride
        words64 = 4 * B + (3 * B + 1) // 2 if KF == 0 else (B * KF * 5 + 4 * B + 1) // 2
        self.host = torch.zeros(words64, dtype=torch.int64)
        if torch.cuda.is_available():
            self.host = self.host.pin_memory()
        self.dev = torch.zeros(words64, dtype=torch.int64, device=self.device)
        self.image_wh = None            # (W, H) of the per-object keyframe images (per-object mode)
        self._uploaded = None           # event recorded after the last host->device copy of the pinned buffer

    def _wait_upload(self) -> None:
        """The pinned buffer may still be the source of an in-flight (asynchronous) upload of the previous frame:
        wait for that copy -- only the copy, not the frame's kernels -- before overwriting it."""
        if self._uploaded is not None:
            self._uploaded.synchronize()

    def fill_objects(self, sets: Sequence[KeyframeSet]) -> None:
        B = self.n_obj
        assert self.kf_stride == 0 and len(sets) == B
        self._wait_upload()
        for o in sets:
            assert o.rgbs_batch.is_contiguous() and o.depth_batch.is_contiguous()
            assert o.t_wc_batch.is_contiguous() and o.bbox.is_contiguous()
            assert o.rgbs_batch.dtype == torch.uint8 and o.depth_batch.dtype == torch.float32
            assert o.rgbs_batch.device == self.device
        self.image_wh = (int(sets[0].rgbs_batch.shape[1]), int(sets[0].rgbs_batch.shape[2]))
        i32 = [o.n_keyframes for o in sets] + [v for o in sets for v in _latest2(o.latest_kf)]
        if len(i32) & 1:
            i32.append(0)
        cols = ([o.rgbs_batch.data_ptr() for o in sets] + [o.depth_batch.data_ptr() for o in sets] +
                [o.t_wc_batch.data_ptr() for o in sets] + [o.bbox.data_ptr() for o in sets])
        self.host.copy_(torch.tensor(cols + [(i32[k] & 0xffffffff) | (i32[k + 1] << 32) for k in range(0, len(i32), 2)],
                                     dtype=torch.int64))

    def fill_store(self, kt: "KeyframeTables") -> None:
        B, KF = self.n_obj, self.kf_stride
        assert kt.kf_slot.shape == (B, KF)
        self._wait_upload()
        h = self.host.view(torch.int32)
        o = 0
        for t in (kt.kf_slot, kt.kf_bbox.view(torch.int32), kt.obj_id, kt.n_kf, kt.latest):
            h[o:o + t.numel()] = t.reshape(-1)
            o += t.numel()

    def upload(self) -> None:
        self.dev.copy_(self.host, non_blocking=True)
        if self.dev.is_cuda and not torch.cuda.is_current_stream_capturing():
            if self._uploaded is None:
                self._uploaded = torch.cuda.Event()
            self._uploaded.record(torch.cuda.current_stream(self.device))

    def bind(self, a) -> None:
        B, KF = self.n_obj, self.kf_stride
        if KF == 0:
            ptrs = self.dev[:4 * B].view(4, B)
            tail = self.dev[4 * B:].view(torch.int32)
            a.rgbs, a.depths, a.t_wc, a.bbox = _p(ptrs[0]), _p(ptrs[1]), _p(ptrs[2]), _p(ptrs[3])
            a.n_keyframes, a.latest_kf = _p(tail[:B]), _p(tail[B:3 * B])
        else:
            d = self.dev.view(torch.int32)
            o1 = B * KF
            o2 = o1 + B * KF * 4
            a.kf_slot, a.kf_bbox, a.obj_id, a.kf_stride = _p(d[:o1]), _p(d[o1:o2]), _p(d[o2:o2 + B]), KF
            a.n_keyframes, a.latest_kf = _p(d[o2 + B:o2 + 2 * B]), _p(d[o2 + 2 * B:o2 + 4 * B])


def _latest2(q):
    q = list(q)
    return q[-2:] if len(q) >= 2 else [q[0] if q else 0] * 2


class KeyframeTables:
    """Host-side per-object keyframe tables of the shared store, packed into ONE pinned buffer so a frame's
    sampling needs a single small host->device copy (instead of B x 4 pointer-table entries)."""

    def __init__(self, kf_slot, kf_bbox, obj_id, n_kf, latest):
        self.kf_slot = torch.as_tensor(kf_slot, dtype=torch.int32).contiguous()          # [B,KF]
        self.kf_bbox = torch.as_tensor(kf_bbox, dtype=torch.float32).contiguous()        # [B,KF,4]
        self.obj_id = torch.as_tensor(obj_id, dtype=torch.int32).contiguous()            # [B]
        self.n_kf = torch.as_tensor(n_kf, dtype=torch.int32).contiguous()                # [B]
        self.latest = torch.as_tensor(latest, dtype=torch.int32).contiguous()            # [B,2]
        B, KF = self.kf_slot.shape
        assert self.kf_bbox.shape == (B, KF, 4) and self.obj_id.shape == (B,) and self.latest.shape == (B, 2)
