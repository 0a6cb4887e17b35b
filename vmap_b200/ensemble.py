"""Packed ensemble state + the fused training step (the package's public step API).

One ``VmapEnsemble`` owns, for a stack of ``n_obj`` object MLPs on one GPU:
``params | grads | exp_avg | exp_avg_sq`` as ``[n_obj, stride]`` fp32 blocks, the fp16
tensor-core weight image, per-object scales, loss terms and the status word.  It replaces
what ``utils.update_vmap`` + ``torch.optim.AdamW`` hold in the reference
(utils.py:30-34, train.py:67) and runs train.py:293-326 as ONE kernel launch at hidden 32 (mask counts, fused
forward+loss+backward, ordered gradient reduction and AdamW all inside ``vmb_step(fuse_adam=1)``); wide models
(hidden 64/128/256) run mask counts + the layer-wise step + the AdamW kernel behind the same call.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
from typing import Dict, Optional

import torch

from . import _lib
from .layout import ALL_KEYS, host_offsets, tensor_shapes


class LossExplode(RuntimeError):
    """The reference prints 'loss explode' and exit(-1)s (render_rays.py:88-90);
    here the update is skipped on the device and this is raised at the next check."""


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def rows_dense(t: torch.Tensor) -> bool:
    """True when every t[i] is a dense block (what ``t[i].is_contiguous()`` says, without building the view)."""
    expect = 1
    shape, stride = t.shape, t.stride()
    for d in range(t.dim() - 1, 0, -1):
        if shape[d] != 1 and stride[d] != expect:
            return False
        expect *= shape[d]
    return True


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class VmapEnsemble:
    def __init__(self, n_obj: int, hidden: int = 32, n_unidir_funcs: int = 5, scale=2.0,
                 device="cuda:0", lr: float = 1e-3, weight_decay: float = 0.013,
                 betas=(0.9, 0.999), eps: float = 1e-8, impl: str = "auto",
                 colour_scaling: float = 5.0, opacity_scaling: float = 10.0):
        self.lib = _lib.lib()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.VmbError("VmapEnsemble needs a CUDA device: there is no CPU fallback")
        self.n_obj, self.hidden, self.n_unidir_funcs = n_obj, hidden, n_unidir_funcs
        self.n_freq = n_unidir_funcs + 1
        self.lr, self.weight_decay, self.betas, self.eps = lr, weight_decay, betas, eps
        # VMB_IMPL=fp32|umma|layerwise overrides the default choice ("auto"), e.g. to run the drop-in on the fp32 parity kernel
        self.impl = os.environ.get("VMB_IMPL", impl) if impl == "auto" else impl
        self.colour_scaling, self.opacity_scaling = colour_scaling, opacity_scaling
        self.count, self.stride, self.offsets, self.sizes = _lib.param_layout(hidden, self.n_freq)
        assert (self.count, self.stride, self.offsets, self.sizes) == host_offsets(hidden, n_unidir_funcs)
        self.shapes = tensor_shapes(hidden, n_unidir_funcs)
        dev = self.device
        with torch.cuda.device(dev):
            self._handle = C.c_void_p()
            _lib.check(None, self.lib.vmb_create(C.byref(self._handle), dev.index or 0, n_obj, hidden, self.n_freq),
                       "vmb_create")
        f32 = dict(dtype=torch.float32, device=dev)
        self.params = torch.zeros(n_obj, self.stride, **f32)
        self.grads = torch.zeros(n_obj, self.stride, **f32)
        self.exp_avg = torch.zeros(n_obj, self.stride, **f32)
        self.exp_avg_sq = torch.zeros(n_obj, self.stride, **f32)
        self.image_bytes = self.lib.vmb_image_bytes(hidden, self.n_freq)
        self.image = torch.zeros(n_obj, self.image_bytes, dtype=torch.uint8, device=dev) if self.image_bytes else None
        sc = torch.as_tensor(scale, dtype=torch.float32)
        self.scale = (sc.expand(n_obj) if sc.dim() == 0 else sc).to(dev).contiguous().clone()
        self.loss_terms = torch.zeros(n_obj, 4, **f32)
        self.status = torch.zeros(4, dtype=torch.int32, device=dev)
        self._grad_scale = self._grad_scale_held = None
        self.loss_calls = 0                                 # step_batch_loss launches so far (their slot in loss_ring)
        self.loss_ring = torch.zeros(4096, **f32)          # scalar loss of step t (sum over objects) lands in slot t % 4096
        self.step_count = 0
        # per-object step numbers on the device: graph replay needs them there, and objects that join a stack later
        # (update_vmap(..., keep_optimizer_state=True)) keep their own bias correction
        self.step_counter = torch.zeros(n_obj, dtype=torch.int32, device=dev)

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self.lib.vmb_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    # ---- stacked views (what update_vmap returns as `params`, utils.py:31) ---------------
    def view(self, key: str, block: Optional[torch.Tensor] = None) -> torch.Tensor:
        i = ALL_KEYS.index(key)
        blk = self.params if block is None else block
        return blk[:, self.offsets[i]:self.offsets[i] + self.sizes[i]].view((self.n_obj,) + self.shapes[key])

    def stacked(self, block: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        return {k: self.view(k, block) for k in ALL_KEYS}

    def load_stacked(self, tensors: Dict[str, torch.Tensor], reset_optimizer: bool = True):
        """Copy stacked [n_obj, *shape] tensors in.  ``reset_optimizer`` reproduces the
        reference's behaviour of starting Adam from scratch whenever update_vmap
        re-stacks (SURVEY.md 3.4)."""
        with torch.no_grad():
            for k in ALL_KEYS:
                self.view(k).copy_(tensors[k].to(self.device, torch.float32))
        if reset_optimizer:
            self.reset_optimizer()
        self.refresh_image()

    def reset_optimizer(self):
        self.exp_avg.zero_(); self.exp_avg_sq.zero_(); self.grads.zero_()
        self.step_count = 0
        self.step_counter.zero_()

    def reset_optimizer_row(self, row: int):
        """Start AdamW from scratch for ONE object (a freshly loaded checkpoint, vmap.py:478-491)."""
        self.exp_avg[row].zero_(); self.exp_avg_sq[row].zero_(); self.grads[row].zero_()
        self.step_counter[row] = 0

    def refresh_image(self):
        if self.image is not None:
            with torch.cuda.device(self.device):
                _lib.check(self._handle, self.lib.vmb_build_image(self._handle, self.n_obj, _ptr(self.params),
                                                                  _ptr(self.image), _stream()), "vmb_build_image")

    def _on_device(self):
        """Context that makes ``self.device`` current; free when it already is (the common single-GPU case)."""
        if torch.cuda.current_device() == self.device.index:
            return contextlib.nullcontext()
        return torch.cuda.device(self.device)

    # ---- kernels ----------------------------------------------------------------------------
    def _step_args(self, batch, backward: bool, outputs=None, impl: Optional[str] = None, counts=None,
                   fuse_adam: bool = False, guard_loss: bool = True, loss_out: Optional[torch.Tensor] = None):
        pcs, z = batch["pcs"], batch["z"]
        B, R, S = pcs.shape[0], pcs.shape[1], pcs.shape[2]
        assert B == self.n_obj and pcs.shape[3] == 3 and tuple(z.shape) == (B, R, S)
        gd, gc, sem, md = batch["gt_depth"], batch["gt_colour"], batch["sem"], batch["mask_depth"]
        for t, dt in ((pcs, torch.float32), (z, torch.float32), (gd, torch.float32), (gc, torch.float32)):
            assert t.dtype == dt and t.device == self.device
        assert sem.dtype == torch.uint8 and md.dtype in (torch.bool, torch.uint8)
        # per-object slices of a bigger tensor are fine as long as each object's block is dense
        for t in (pcs, z, gd, gc, sem, md):
            assert rows_dense(t), "per-object block must be contiguous"
        a = _lib.StepArgs()
        a.n_obj, a.n_rays, a.n_samples = B, R, S
        a.impl = _lib.VMB_IMPL[impl or self.impl]
        a.pcs, a.pcs_stride = _ptr(pcs), pcs.stride(0) if B > 1 else R * S * 3
        a.z_vals, a.z_stride = _ptr(z), z.stride(0) if B > 1 else R * S
        a.gt_depth, a.gt_depth_stride = _ptr(gd), gd.stride(0) if B > 1 else R
        a.gt_colour, a.gt_colour_stride = _ptr(gc), gc.stride(0) if B > 1 else R * 3
        a.sem, a.sem_stride = _ptr(sem), sem.stride(0) if B > 1 else R
        a.mask_depth, a.mask_stride = _ptr(md), md.stride(0) if B > 1 else R
        a.params, a.image, a.scale = _ptr(self.params), _ptr(self.image), _ptr(self.scale)
        a.grads, a.loss_terms = _ptr(self.grads), _ptr(self.loss_terms)
        if outputs is not None:
            a.r_depth, a.r_var = _ptr(outputs["depth"]), _ptr(outputs["var"])
            a.r_colour, a.r_opacity = _ptr(outputs["colour"]), _ptr(outputs["opacity"])
        a.counts = _ptr(counts)
        a.colour_scaling, a.opacity_scaling = self.colour_scaling, self.opacity_scaling
        a.backward = 1 if backward else 0
        if loss_out is not None:
            assert loss_out.dtype == torch.float32 and loss_out.device == self.device and loss_out.numel() >= 1
            a.loss_sum = _ptr(loss_out)
        if fuse_adam:
            a.fuse_adam = 1
            a.exp_avg, a.exp_avg_sq = _ptr(self.exp_avg), _ptr(self.exp_avg_sq)
            a.step_counter, a.step = _ptr(self.step_counter), 0
            a.lr, a.beta1, a.beta2, a.eps = self.lr, self.betas[0], self.betas[1], self.eps
            a.weight_decay = self.weight_decay
            a.guard_loss, a.status = (1 if guard_loss else 0), _ptr(self.status)
        return a

    def forward_backward(self, batch, outputs=None, backward: bool = True, impl: Optional[str] = None,
                         counts: Optional[torch.Tensor] = None, k1_events=None, fuse_adam: bool = False,
                         guard_loss: bool = True, loss_out: Optional[torch.Tensor] = None):
        """K0 + K1: accumulates into ``self.grads`` and overwrites ``self.loss_terms``; with ``fuse_adam`` the
        optimiser update happens in the same call (``self.grads`` untouched at hidden 32).
        ``k1_events`` = (start, stop) torch.cuda.Event pair recorded around the K1 launch."""
        a = self._step_args(batch, backward, outputs, impl, counts, fuse_adam, guard_loss, loss_out)
        if k1_events is not None:
            for ev in k1_events:
                if not ev.cuda_event:
                    ev.record()                  # torch creates the CUDA event lazily
            a.k1_start_event = C.c_void_p(k1_events[0].cuda_event)
            a.k1_stop_event = C.c_void_p(k1_events[1].cuda_event)
        with self._on_device():
            _lib.check(self._handle, self.lib.vmb_step(self._handle, C.byref(a), _stream()), "vmb_step")

    def mask_counts(self, batch) -> torch.Tensor:
        sem, md = batch["sem"], batch["mask_depth"]
        B, R = sem.shape
        out = torch.empty(B, 4, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._handle, self.lib.vmb_mask_counts(
                self._handle, B, R, _ptr(sem), sem.stride(0) if B > 1 else R,
                _ptr(md), md.stride(0) if B > 1 else R, _ptr(out), _stream()), "vmb_mask_counts")
        return out

    def adam_step(self, guard_loss: bool = True, device_counter: bool = True):
        """K2: AdamW over the whole block + zero_grad (+ fp16 image refresh).  With
        ``device_counter`` the step number lives on the device (incremented by the kernel),
        which is what makes a captured CUDA graph of the step replayable."""
        self.step_count += 1
        a = _lib.AdamArgs()
        a.n_obj, a.step = self.n_obj, (0 if device_counter else self.step_count)
        a.step_counter = _ptr(self.step_counter) if device_counter else None
        a.params, a.grads = _ptr(self.params), _ptr(self.grads)
        a.exp_avg, a.exp_avg_sq = _ptr(self.exp_avg), _ptr(self.exp_avg_sq)
        a.image = _ptr(self.image)
        a.loss_terms = _ptr(self.loss_terms) if guard_loss else None
        a.status = _ptr(self.status)
        a.lr, a.beta1, a.beta2, a.eps = self.lr, self.betas[0], self.betas[1], self.eps
        a.weight_decay, a.zero_grads = self.weight_decay, 1
        if self._grad_scale is not None:                      # upstream gradient of loss.backward(), applied by the kernel
            a.grad_scale = _ptr(self._grad_scale)
        self._grad_scale_held, self._grad_scale = self._grad_scale, None     # keep it alive past the asynchronous launch
        with self._on_device():
            _lib.check(self._handle, self.lib.vmb_adam(self._handle, C.byref(a), _stream()), "vmb_adam")

    def step(self, batch, impl: Optional[str] = None, loss_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One optimisation step (train.py:293-326) in one library call.  Returns the summed loss as a device scalar
        with no reduction launch on the Python side: the step kernel's last CTA writes it into ``loss_out`` (a float32
        device tensor) or, by default, into the next slot of a 4096-entry ring (so returned scalars stay valid -- and
        distinct -- for the next 4095 steps; ``.item()`` / ``.clone()`` them to keep them longer)."""
        if loss_out is None:
            slot = self.step_count % self.loss_ring.numel()
            loss_out = self.loss_ring[slot:slot + 1]
        self.forward_backward(batch, impl=impl, fuse_adam=True, loss_out=loss_out)
        self.step_count += 1
        return loss_out.view(-1)[0]

    def joint_step(self, batch, ba_args, group: int = 0, loss_out: Optional[torch.Tensor] = None, outputs=None,
                   pcs_world_out: Optional[torch.Tensor] = None) -> None:
        """The step of one joint map-and-pose iteration (``vmb_joint_step_lw``, hidden 64/128/256): ``batch["pcs"]``
        holds camera-frame points, moved to the world by the pose of each ray's draw (``ba_args``: the fp64 pose table
        and, in ``group``, the draw layout, keyframe tables and ray rows); the layer-wise step on those points
        accumulates into ``self.grads`` and overwrites ``self.loss_terms`` (``loss_out`` / ``outputs`` as in
        ``step`` / ``render``), and the step's own embedding gradient gives the per-ray pose rows.  No optimiser update:
        ``adam_step`` and ``vmb_ba_update`` follow.  ``pcs_world_out``: [B,R,S,3] float32 copy of the world points."""
        a = self._step_args(batch, True, outputs, "layerwise", loss_out=loss_out)
        if pcs_world_out is not None:
            assert pcs_world_out.shape == batch["pcs"].shape and pcs_world_out.is_contiguous()
            assert pcs_world_out.dtype == torch.float32 and pcs_world_out.device == self.device
        with self._on_device():
            _lib.check(self._handle, self.lib.vmb_joint_step_lw(self._handle, C.byref(a), C.byref(ba_args), group,
                                                                _ptr(pcs_world_out), _stream()), "vmb_joint_step_lw")

    def joint_step_fused(self, batch, ba_args, group: int = 0, fuse_adam: bool = True,
                         loss_out: Optional[torch.Tensor] = None, outputs=None,
                         pcs_world_out: Optional[torch.Tensor] = None) -> None:
        """The step of one joint map-and-pose iteration at hidden 32 (``vmb_joint_step_fused``): as ``joint_step``, on the
        fused hidden-32 step, whose PE backward also gives every point's pose gradient.  ``fuse_adam`` (default): AdamW
        runs inside the step, as ``step`` does (the pose terms read the directions before it); otherwise the gradients
        accumulate into ``self.grads`` for ``adam_step``.  ``vmb_ba_update`` follows."""
        a = self._step_args(batch, True, outputs, "umma", fuse_adam=fuse_adam, loss_out=loss_out)
        if pcs_world_out is not None:
            assert pcs_world_out.shape == batch["pcs"].shape and pcs_world_out.is_contiguous()
            assert pcs_world_out.dtype == torch.float32 and pcs_world_out.device == self.device
        with self._on_device():
            _lib.check(self._handle, self.lib.vmb_joint_step_fused(self._handle, C.byref(a), C.byref(ba_args), group,
                                                                   _ptr(pcs_world_out), _stream()),
                       "vmb_joint_step_fused")
        if fuse_adam:
            self.step_count += 1

    def capture_step(self, batch, impl: Optional[str] = None) -> "torch.cuda.CUDAGraph":
        """Capture the step (one launch at hidden 32) on ``batch``'s (fixed) buffers into a CUDA graph; refill the buffers
        and ``replay()`` for every step.  Removes the per-launch host overhead of the loop."""
        self.forward_backward(batch, impl=impl, backward=False)      # warm-up: sets kernel attributes
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.forward_backward(batch, impl=impl, fuse_adam=True)
        self._graph_batch = batch
        return g

    def render(self, batch, impl: Optional[str] = None):
        """Forward + render only: (depth [B,R], var [B,R], colour [B,R,3], opacity [B,R])."""
        B, R = batch["gt_depth"].shape
        f32 = dict(dtype=torch.float32, device=self.device)
        out = {"depth": torch.empty(B, R, **f32), "var": torch.empty(B, R, **f32),
               "colour": torch.empty(B, R, 3, **f32), "opacity": torch.empty(B, R, **f32)}
        self.forward_backward(batch, outputs=out, backward=False, impl=impl)
        return out["depth"], out["var"], out["colour"], out["opacity"]

    def eval_points(self, points: torch.Tensor, impl: Optional[str] = None, row: Optional[int] = None,
                    chunk: int = 1 << 21, out=None):
        """Forward only on raw points -> alpha (raw*10, model.py:77), colour (trainer.py:77-90).
        ``row=None``: points [B,N,3], every object evaluates its own set -> alpha [B,N], colour [B,N,3].
        ``row=r``: points [N,3] evaluated by object r ONLY (one-row views of the packed state are handed to
        ``vmb_forward`` with n_obj = 1, so meshing one object of a 160-object stack costs one object's work)
        -> alpha [N], colour [N,3].  ``chunk`` bounds the points per launch (the reference uses 100k chunks).
        ``impl="fp32"`` forces the CUDA-core kernel; otherwise hidden 32 runs the forward half of the fused
        wgmma kernel and hidden 64/128/256 the layer-wise wgmma GEMMs, on the fp16 weight image.
        ``out=(alpha, colour)``: contiguous fp32 device tensors of the result's shape to write into (and return)."""
        if row is None:
            B, N, _ = points.shape
            assert B == self.n_obj
            params, scale, image = self.params, self.scale, self.image
        else:
            assert 0 <= row < self.n_obj and points.dim() == 2
            B, N = 1, points.shape[0]
            points = points[None]
            params, scale = self.params[row:row + 1], self.scale[row:row + 1]
            image = self.image[row:row + 1] if self.image is not None else None
        assert points.is_contiguous() and points.dtype == torch.float32 and points.device == self.device
        if out is None:
            alpha = torch.empty(B, N, dtype=torch.float32, device=self.device)
            colour = torch.empty(B, N, 3, dtype=torch.float32, device=self.device)
        else:
            alpha, colour = out[0].view(B, N), out[1].view(B, N, 3)
            for t in (alpha, colour):
                assert t.is_contiguous() and t.dtype == torch.float32 and t.device == self.device
        use_image = (impl or self.impl) != "fp32" and image is not None
        with torch.cuda.device(self.device):
            for n0 in range(0, N, chunk):
                n = min(chunk, N - n0)
                a = _lib.ForwardArgs()
                a.n_obj, a.n_points = B, n
                a.points, a.points_stride = C.c_void_p(points.data_ptr() + n0 * 12), N * 3
                a.params, a.scale = _ptr(params), _ptr(scale)
                a.alpha, a.alpha_stride = C.c_void_p(alpha.data_ptr() + n0 * 4), N
                a.colour, a.colour_stride = C.c_void_p(colour.data_ptr() + n0 * 12), N * 3
                if use_image:
                    a.image = _ptr(image)
                _lib.check(self._handle, self.lib.vmb_forward(self._handle, C.byref(a), _stream()), "vmb_forward")
        if row is not None:
            return alpha[0], colour[0]
        return alpha, colour

    def poll_status(self):
        """Asynchronous guard (no host sync): copy the device status word to pinned memory after this step's
        work and raise if a copy enqueued by an EARLIER call has landed with a guard bit set.  The reference
        exit(-1)s on a loss explosion (render_rays.py:88-90); here the device skips the update and training
        stops with LossExplode at most one poll later.  Called by FusedAdamW.step and FrameLoop.run."""
        if getattr(self, "_status_host", None) is None:
            self._status_host = torch.zeros(4, dtype=torch.int32).pin_memory()
            self._status_event = torch.cuda.Event()
            self._status_pending = False
        if self._status_pending and self._status_event.query():
            self._raise_for(int(self._status_host[0]))
        if torch.cuda.is_current_stream_capturing():
            return
        self._status_host.copy_(self.status, non_blocking=True)
        self._status_event.record(torch.cuda.current_stream(self.device))
        self._status_pending = True

    @staticmethod
    def _raise_for(st: int):
        if st & _lib.VMB_ST_LOSS_EXPLODE:
            raise LossExplode("loss explode (a per-object loss term exceeded 1e5); update skipped")
        if st & _lib.VMB_ST_NONFINITE:
            raise LossExplode("non-finite loss; update skipped")

    def check_status(self):
        """Host sync: raise if the device flagged a loss explosion / non-finite loss."""
        self._raise_for(int(self.status[0].item()))


class StepInputs:
    """One flat byte buffer holding the six input tensors of a step, so that a step's inputs
    move host->device with a single copy (pinned twin on the host side)."""

    FIELDS = (("pcs", torch.float32, lambda B, R, S: (B, R, S, 3)), ("z", torch.float32, lambda B, R, S: (B, R, S)),
              ("gt_depth", torch.float32, lambda B, R, S: (B, R)), ("gt_colour", torch.float32, lambda B, R, S: (B, R, 3)),
              ("sem", torch.uint8, lambda B, R, S: (B, R)), ("mask_depth", torch.uint8, lambda B, R, S: (B, R)))

    def __init__(self, n_obj: int, n_rays: int, n_samples: int, device="cpu", pinned: bool = False):
        off, spans = 0, []
        for name, dt, shp in self.FIELDS:
            shape = shp(n_obj, n_rays, n_samples)
            nbytes = torch.empty((), dtype=dt).element_size()
            for d in shape:
                nbytes *= d
            spans.append((name, dt, shape, off, nbytes))
            off = (off + nbytes + 255) // 256 * 256
        self.nbytes = off
        self.flat = torch.empty(off, dtype=torch.uint8, device=device)
        if pinned:
            self.flat = self.flat.pin_memory()
        self.views: Dict[str, torch.Tensor] = {
            name: self.flat[o:o + n].view(dt).view(shape) for name, dt, shape, o, n in spans}
        self.payload_bytes = sum(n for *_, n in spans)

    def fill(self, batch: Dict[str, torch.Tensor]):
        for k, v in self.views.items():
            v.copy_(batch[k].to(v.dtype))
        return self

    def copy_from(self, other: "StepInputs", non_blocking: bool = True):
        self.flat.copy_(other.flat, non_blocking=non_blocking)
        return self
