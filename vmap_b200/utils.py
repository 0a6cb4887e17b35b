"""utils.update_vmap with the reference's signature (utils.py:30-34), the ``vmap`` shim
that replaces ``functorch.vmap`` at train.py:293-294, the picklable ``BoundingBox`` that
sceneObject.get_bound stores in checkpoints (utils.py:11-24), and ``capture_graph``, the warm-up and capture of the
package's CUDA-graph loops (mapping frames, tracking, bundle adjustment)."""
from __future__ import annotations

import torch

from .layout import FC_KEYS, PE_KEY
from .lazy import LazyEmbedding, LazyHeads, bind_modules


class BoundingBox:
    """Oriented 3-D box (utils.py:11-18): ``center`` [3], ``R`` [3,3] (box axes as columns), ``extent`` [3]."""

    def __init__(self):
        self.extent = None
        self.R = None
        self.center = None
        self.points3d = None    # (8,3)


def bbox_open3d2bbox(bbox_o3d):
    """utils.py:20-25: anything with .extent / .R / .center -> BoundingBox."""
    bbox = BoundingBox()
    bbox.extent = bbox_o3d.extent
    bbox.R = bbox_o3d.R
    bbox.center = bbox_o3d.center
    return bbox


class _Stack:
    """What one optimiser's two update_vmap calls (fc, then pe) build together."""

    def __init__(self):
        self.fc, self.pe, self.ens = None, None, None
        self.keep_state = False

    def maybe_build(self):
        from .ensemble import VmapEnsemble
        if not self.fc or not self.pe or len(self.fc) != len(self.pe):
            return
        fc0, pe0 = self.fc[0], self.pe[0]
        dev = next(fc0.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("update_vmap: models must be on a CUDA device (there is no CPU path)")
        # re-stacking starts AdamW from scratch for every object, as the reference does
        # (fresh leaves + a new param group, utils.py:31-33; SURVEY.md 3.4) -- unless the caller opted in to
        # keep_optimizer_state (SURVEY.md 8(f)3): objects already training keep their Adam moments AND their own
        # step number (per-object bias correction), only the newcomers start from zero
        old = [getattr(fc, "_vmb_binding", None) for fc in self.fc] if self.keep_state else []
        old = [(b[0](), b[1]) if b is not None and b[0]() is not None else None for b in old]
        ens = VmapEnsemble(len(self.fc), hidden=fc0.hidden_size, n_unidir_funcs=pe0.max_deg,
                           scale=[float(p.scale) for p in self.pe], device=dev)
        for i, (fc, pe) in enumerate(zip(self.fc, self.pe)):
            bind_modules(ens, i, fc, pe)
        for i, o in enumerate(old):
            if o is not None and o[0].stride == ens.stride:
                ens.exp_avg[i].copy_(o[0].exp_avg[o[1]])
                ens.exp_avg_sq[i].copy_(o[0].exp_avg_sq[o[1]])
                ens.step_counter[i] = o[0].step_counter[o[1]]
        ens.refresh_image()
        self.ens = ens


class FusedModel:
    def __init__(self, kind, stack):
        self.kind, self.stack = kind, stack

    def batched(self, params, buffers, x):
        if self.stack.ens is None:
            raise RuntimeError("update_vmap must be called for both the fc and the pe models first")
        if self.kind == "pe":
            return LazyEmbedding(x, ens=self.stack.ens)
        heads = LazyHeads(x)
        return heads.alpha, heads.color


class StackedParams:
    """``params[i][model_id]`` as used by train.py:335-338: stacked [n_obj, *shape] views."""

    def __init__(self, kind, stack):
        self.keys = FC_KEYS if kind == "fc" else (PE_KEY,)
        self.stack = stack

    def __len__(self):
        return len(self.keys)

    def __getitem__(self, i):
        return self.stack.ens.view(self.keys[i])

    def __iter__(self):
        return (self[i] for i in range(len(self)))


class StackedBuffers(StackedParams):
    def __init__(self, kind, stack):
        self.keys = () if kind == "fc" else ("scale",)
        self.stack = stack

    def __getitem__(self, i):
        return self.stack.ens.scale


def update_vmap(models, optimiser, keep_optimizer_state=False):
    """(fmodel, params, buffers) for a list of per-object modules; call once for the
    OccupancyMaps and once for the UniDirsEmbeds (train.py:181-182).
    ``keep_optimizer_state=True`` (opt-in deviation from utils.py:30-34, where every re-stack silently resets
    AdamW): modules that were already bound to a stack carry their exp_avg / exp_avg_sq rows and step number over."""
    from .model import OccupancyMap
    stack = optimiser.__dict__.setdefault("_vmb_stack", _Stack())
    stack.keep_state = stack.keep_state or bool(keep_optimizer_state)
    kind = "fc" if isinstance(models[0], OccupancyMap) else "pe"
    setattr(stack, kind, list(models))
    stack.maybe_build()
    params = StackedParams(kind, stack)
    optimiser.add_param_group({"params": [], "vmb_stack": kind})
    return FusedModel(kind, stack), params, StackedBuffers(kind, stack)


def vmap(fmodel, *args, **kwargs):
    """Drop-in for ``functorch.vmap`` at train.py:293-294."""
    if not isinstance(fmodel, FusedModel):
        raise TypeError("vmap_b200.vmap only maps the fused models returned by update_vmap "
                        "(no tracing / PyTorch fallback)")
    return fmodel.batched


def capture_graph(device, enqueue, keep) -> torch.cuda.CUDAGraph:
    """One CUDA graph of ``enqueue``: a warm-up call ``enqueue(upload=True)`` on a side stream (kernel attributes, the
    allocator's pools), a synchronise, then the capture of ``enqueue(upload=False)``.  The tensors in ``keep`` get back
    the values they had before the warm-up, so neither run leaves a trace in them."""
    snap = [t.clone() for t in keep]
    st = torch.cuda.Stream(device=device)
    st.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(st):
        enqueue(upload=True)
    torch.cuda.current_stream(device).wait_stream(st)
    torch.cuda.synchronize(device)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        enqueue(upload=False)
    for dst, src in zip(keep, snap):
        dst.copy_(src)
    return graph


def box_filter(masks, classes, depth, inst_dict, intrinsic_open3d, T_CW, min_pixels=500, voxel_size=0.01):
    """utils.box_filter (utils.py:112-208) with the reference's signature and return value (int64 [H, W]), run by
    the GPU instance tracker of vmap_b200.scannet; the tracking state follows the ``inst_dict`` object."""
    from .scannet import box_filter as _box_filter
    return _box_filter(masks, classes, depth, inst_dict, intrinsic_open3d, T_CW, min_pixels, voxel_size)
