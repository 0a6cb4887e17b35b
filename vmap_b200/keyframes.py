"""Shared keyframe store + GPU frame ingest (SURVEY.md 8(f) rows 2 and 4).

The reference gives every object its own full-frame copies of each of its keyframes
(``sceneObject.rgbs_batch`` / ``depth_batch``, vmap.py:137-176: ~130 MB per object at
20 x 1200 x 680) and, per new frame, builds one uint8 state image per visible object on the
data device (train.py:121-128) before copying the frame into each object's buffers
(train.py:135-141 -> vmap.py:208-263).  Here a frame is stored ONCE in a ``FrameStore`` slot
(rgb, depth, pose and the instance image); objects keep ``(store slot, bbox)`` tables and the
sampler derives the pixel state from the instance id.  ``FrameStore.ingest`` is the GPU pass
that replaces the per-frame numpy loop of dataset.py:101-131 (unique ids, one boolean mask per
instance, ``get_bbox2d_batch``, ``enlarge_bbox``, background relabel).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import torch

from . import _lib

STAT_COLS = ("count", "u_min", "u_max1", "v_min", "v_max1", "cls_min", "cls_max", "keep")


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class FrameStore:
    """Fixed-capacity pool of posed RGB-D + instance frames on one GPU, reference counted.

    ``put``/``ingest`` return a slot holding one reference (the caller's); every keyframe-table entry
    of an object that points at the slot holds another.  A slot returns to the free list when the last
    reference is released, so frames no object kept cost nothing after ``release``.
    """

    def __init__(self, width: int, height: int, capacity: int, device="cuda:0", max_id: int = 4096):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.VmbError("FrameStore lives in GPU memory: there is no CPU fallback")
        self.lib = _lib.lib()
        self.W, self.H, self.capacity, self.max_id = width, height, capacity, max_id
        dev = self.device
        self.rgbx = torch.zeros(capacity, width, height, 4, dtype=torch.uint8, device=dev)
        self.depth = torch.zeros(capacity, width, height, dtype=torch.float32, device=dev)
        self.inst = torch.zeros(capacity, width, height, dtype=torch.int32, device=dev)
        self.t_wc = torch.zeros(capacity, 4, 4, dtype=torch.float32, device=dev)
        self.refcount = [0] * capacity
        self.frame_id: Dict[int, object] = {}
        self._free = list(range(capacity - 1, -1, -1))
        self._handle = C.c_void_p()
        with torch.cuda.device(dev):
            _lib.check(None, self.lib.vmb_create(C.byref(self._handle), dev.index or 0, 1, 32, 6), "vmb_create")
        self.stats = torch.zeros(max_id, len(STAT_COLS), dtype=torch.int32, device=dev)
        self.bbox = torch.zeros(max_id, 4, dtype=torch.float32, device=dev)
        self._keep = None

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self.lib.vmb_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    # ---- slots ----------------------------------------------------------------------------------
    @property
    def bytes_per_frame(self) -> int:
        return self.W * self.H * (4 + 4 + 4) + 64

    @property
    def n_used(self) -> int:
        return self.capacity - len(self._free)

    def _take(self, frame_id) -> int:
        if not self._free:
            raise _lib.VmbError(f"FrameStore full ({self.capacity} frames): raise the capacity or release frames")
        s = self._free.pop()
        self.refcount[s] = 1
        self.frame_id[s] = frame_id
        return s

    def acquire(self, slot: int) -> None:
        assert self.refcount[slot] > 0, "acquire of a free slot"
        self.refcount[slot] += 1

    def release(self, slot: int) -> None:
        assert self.refcount[slot] > 0, "release of a free slot"
        self.refcount[slot] -= 1
        if self.refcount[slot] == 0:
            self.frame_id.pop(slot, None)
            self._free.append(slot)

    def grow(self, capacity: int) -> None:
        """Raise the capacity to ``capacity`` slots, keeping every stored frame in its slot.  The frame tensors are
        reallocated, so a CUDA graph captured on this store reads freed memory afterwards: capture again."""
        old = self.capacity
        if capacity <= old:
            return
        extra = capacity - old
        with torch.no_grad():
            for name in ("rgbx", "depth", "inst", "t_wc"):
                t = getattr(self, name)
                setattr(self, name, torch.cat([t, torch.zeros((extra,) + t.shape[1:], dtype=t.dtype, device=t.device)]))
        self.refcount += [0] * extra
        self._free = list(range(capacity - 1, old - 1, -1)) + self._free
        self.capacity = capacity

    # ---- writes ---------------------------------------------------------------------------------
    def put(self, rgb: torch.Tensor, depth: torch.Tensor, inst: torch.Tensor, t_wc: torch.Tensor, frame_id=None) -> int:
        """Store a frame whose instance image is already final (no ingest pass)."""
        s = self._take(frame_id)
        self.rgbx[s, :, :, :3] = rgb.to(self.device)
        self.depth[s] = depth.to(self.device)
        self.inst[s] = inst.to(self.device, torch.int32)
        self.t_wc[s] = t_wc.to(self.device)
        return s

    def ingest(self, rgb: torch.Tensor, depth: torch.Tensor, inst: torch.Tensor, t_wc: torch.Tensor, frame_id=None,
               cls: Optional[torch.Tensor] = None, background_cls: Sequence[int] = (), bbox_scale: float = 0.2,
               min_extent: int = 10, store: bool = True):
        """One GPU pass over a new frame (dataset.py:101-131 + train.py:121-128).

        Returns ``(slot, stats, bbox)``: ``stats [max_id, 8] int32`` (columns ``STAT_COLS``; ``keep`` = the
        instance survives the background-class / size filter), ``bbox [max_id, 4] f32`` enlarged boxes in
        sceneObject order [u_lo, u_hi, v_lo, v_hi]; both stay on the GPU (read ``keep`` rows on the host once
        per frame to create objects).  With ``store`` the frame is written into a slot with dropped
        instances relabelled 0, as the data loader does (dataset.py:128)."""
        dev = self.device
        rgb = rgb.to(dev).contiguous(); depth = depth.to(dev, torch.float32).contiguous()
        inst = inst.to(dev, torch.int32).contiguous()
        assert inst.shape == (self.W, self.H) and depth.shape == (self.W, self.H) and rgb.shape == (self.W, self.H, 3)
        assert rgb.dtype == torch.uint8
        a = _lib.IngestArgs()
        a.width, a.height, a.inst, a.max_id = self.W, self.H, _p(inst), self.max_id
        a.bbox_scale, a.min_extent = float(bbox_scale), int(min_extent)
        bg = None
        if cls is not None:
            cls = cls.to(dev, torch.int32).contiguous()
            a.cls = _p(cls)
            if len(background_cls):
                n_class = max(int(max(background_cls)) + 1, 1)
                bg = torch.zeros(n_class, dtype=torch.uint8)
                bg[list(background_cls)] = 1
                bg = bg.to(dev)
                a.bg_class, a.n_class = _p(bg), n_class
        a.stats, a.bbox = _p(self.stats), _p(self.bbox)
        slot = -1
        if store:
            slot = self._take(frame_id)
            a.rgb, a.depth = _p(rgb), _p(depth)
            a.dst_rgbx, a.dst_depth, a.dst_inst = _p(self.rgbx[slot]), _p(self.depth[slot]), _p(self.inst[slot])
            self.t_wc[slot] = t_wc.to(dev)
        with torch.cuda.device(dev):
            _lib.check(self._handle, self.lib.vmb_ingest_frame(
                self._handle, C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "vmb_ingest_frame")
        self._keep = (rgb, depth, inst, cls, bg)         # alive until the next call (async launches)
        return slot, self.stats, self.bbox

    def visible_objects(self):
        """Host view of the last ingest: {instance id: bbox tensor [4] (device)} for kept instances
        (the reference's ``bbox_dict``, dataset.py:126,131).  One small device->host read per frame."""
        keep = torch.nonzero(self.stats[:, 7]).flatten().tolist()
        return {int(i): self.bbox[i] for i in keep}
