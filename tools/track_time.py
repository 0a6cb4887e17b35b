"""Time one tracking frame (K10) at the Replica vMAP shape and print one JSON line.

20 hidden-32 objects x 120 rays x 10 samples plus a hidden-128 background x 1200 rays x 14 samples, n_iter 20, on a
synthetic 1200 x 680 frame ingested into a FrameStore.  Reports the sampler time, the per-iteration step time of each
group and of the update, each launched alone (CUDA events over many launches), the whole frame eager (host clock around a synchronised
frame) and as a graph replay, the FLOPs from shapes (forward plus the backward to the inputs, 4 (4H^2 + 220H + 63) per
point) and their share of the H100 SXM fp32 data-sheet rate (67 TFLOP/s), with the card's name and power limit.

``--impl layerwise`` times the tensor-core path for the hidden-128 background (hidden 32 stays on K10); ``--impl fused``
also runs the hidden-32 objects on the fused wgmma tile (``vmb_track_step_fused``).  ``--kernels`` adds, from a
``torch.profiler`` run of its own after the timed ones, the device time per launch of each kernel of one iteration.
``--imap`` times the iMAP shape instead: one hidden-256 scene model, 4800 rays x 14 samples over the full frame."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import vmap_oracle as vo  # noqa: E402
from vmap_b200.cfg import Config, replica_room0_dict  # noqa: E402
from vmap_b200.ensemble import VmapEnsemble  # noqa: E402
from vmap_b200.keyframes import FrameStore  # noqa: E402
from vmap_b200.track import Tracker, _iterate, _step  # noqa: E402

FP32_PEAK = 67e12


def flops_per_point(H):
    return 4 * (4 * H * H + 220 * H + 63)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers still stand; say where the card description went
        return f"unknown ({e})"


def ev_time(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n          # us


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--impl", choices=("fp32", "layerwise", "fused"), default="fp32")
    ap.add_argument("--imap", action="store_true", help="the iMAP shape: one hidden-256 model, 4800 x 14")
    ap.add_argument("--kernels", action="store_true", help="per-kernel device time of one iteration (torch.profiler)")
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "track_time measures the GPU; there is no CPU number"
    dev = "cuda:0"
    cfg = Config(config_dict=replica_room0_dict(imap=args.imap))
    n_iter, n_obj = 20, (0 if args.imap else 20)
    W, H = cfg.W, cfg.H
    g = torch.Generator().manual_seed(0)
    inst = torch.zeros(W, H, dtype=torch.int32)
    for i in range(n_obj):                                  # a 5 x 4 grid of instances over a background
        u0, v0 = (i % 5) * 240 + 20, (i // 5) * 170 + 15
        inst[u0:u0 + 180, v0:v0 + 130] = i + 1
    depth = 1.0 + torch.rand(W, H, generator=g) * 3.0
    rgb = torch.randint(0, 256, (W, H, 3), generator=g, dtype=torch.uint8)
    store = FrameStore(W, H, 2, device=dev, max_id=64)
    slot, _, _ = store.ingest(rgb, depth, inst, torch.eye(4))
    if args.imap:                                           # one scene model over the whole frame (dataset.py:95-96)
        scene = VmapEnsemble(1, hidden=256, scale=cfg.obj_scale, impl="fp32")
        scene.load_stacked(vo.init_params(1, 256, seed=2))
        groups = [(scene, [0])]
    else:
        objs = VmapEnsemble(n_obj, hidden=32, scale=2.0, impl="fp32")
        objs.load_stacked(vo.init_params(n_obj, 32, seed=1))
        bg = VmapEnsemble(1, hidden=128, scale=5.0, impl="fp32")
        bg.load_stacked(vo.init_params(1, 128, seed=2))
        groups = [(objs, list(range(1, n_obj + 1))), (bg, [0])]
    T0 = np.eye(4)
    ids = list(range(n_obj + 1))

    tr = Tracker(groups, cfg, n_iter=n_iter, impl=args.impl)
    tr.track(store, slot, T0, ids=ids)
    torch.cuda.synchronize()
    live = tr._live()
    # sampler: both groups' K3 passes for one frame
    def sample():
        for gi, gr in enumerate(live):
            gr.smp.sample_store(store, gr.tables, n_iter, gr.n_pix, tr.rays_dir, seed=gi, out=gr.out,
                                offset_dev=tr.counter)
    t_sample = ev_time(sample, 50)
    # per-iteration kernels on the sampled buffers
    step_us = {}
    for gi, gr in enumerate(live):
        step_us[f"h{gr.ens.hidden}"] = ev_time(lambda gr=gr, gi=gi: _iterate_one(tr, live, gi), 200)
    f64 = dict(dtype=torch.float64, device=dev)
    pose, adam, losses = torch.eye(4, **f64), torch.zeros(12, **f64), torch.zeros(n_iter, **f64)
    status = torch.zeros(4, dtype=torch.int32, device=dev)
    t_iter = ev_time(lambda: _iterate(live, 1, pose, adam, 0.0, 0.0, losses, status), 200)
    t_update = ev_time(lambda: _update_only(tr, live), 200)
    # whole frame, eager and graph
    reps = 20
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        tr.track(store, slot, T0, ids=ids)
    torch.cuda.synchronize()
    t_eager = (time.perf_counter() - t0) * 1e6 / reps
    tr.capture(store, slot, T0, ids=ids)
    tr.run(store, slot, T0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        tr.run(store, slot, T0)
    torch.cuda.synchronize()
    t_graph = (time.perf_counter() - t0) * 1e6 / reps
    if args.imap:
        pts = {256: cfg.n_per_optim * 14}
        shape = {"scene": f"h256 x {cfg.n_per_optim} rays x 14", "n_iter": n_iter}
    else:
        pts = {32: n_obj * cfg.n_per_optim * 10, 128: cfg.n_per_optim_bg * 14}
        shape = {"objects": f"{n_obj} x h32 x {cfg.n_per_optim} rays x 10",
                 "background": f"h128 x {cfg.n_per_optim_bg} rays x 14", "n_iter": n_iter}
    flop_iter = sum(flops_per_point(h) * n for h, n in pts.items())
    out = {
        "card": card(), "impl": args.impl, "shape": shape,
        "sampler_us": round(t_sample, 2), "step_us": {k: round(v, 2) for k, v in step_us.items()},
        "update_us": round(t_update, 2), "iteration_us": round(t_iter, 2),
        "frame_eager_us": round(t_eager, 1), "frame_graph_us": round(t_graph, 1),
        "gflop_per_iteration": round(flop_iter / 1e9, 3),
        "fp32_share_of_peak_per_iteration": round(flop_iter / (t_iter * 1e-6) / FP32_PEAK, 4),
        "fp32_share_of_peak_frame_graph": round(flop_iter * n_iter / (t_graph * 1e-6) / FP32_PEAK, 4),
    }
    if args.kernels:
        out["kernel_us"] = kernel_times(lambda: _iterate(live, 1, pose, adam, 0.0, 0.0, losses, status), 50)
    print(json.dumps(out))


def kernel_times(fn, n):
    """Device time per launch of each kernel ``fn`` launches (mean over ``n`` calls), from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count:
            out[e.key[:60]] = {"us": round(e.device_time_total / e.count, 2), "launches": e.count}
    return out


def _update_only(tr, live):
    """vmb_track_update alone on the partials iteration 0 left (zero rates: the pose does not move)."""
    import ctypes as C
    from vmap_b200 import _lib
    from vmap_b200.ensemble import _ptr, _stream
    a = _lib.TrackArgs()
    a.n_groups, a.n_iter, a.iter = len(live), tr.n_iter, 1
    a.pose, a.adam = _ptr(tr.pose), _ptr(tr.adam)
    a.beta1, a.beta2, a.eps = 0.9, 0.999, 1e-8
    a.colour_scaling, a.opacity_scaling = 5.0, 10.0
    for k, gr in enumerate(live):
        gr.bind(a.group[k], 0)
    e = live[0].ens
    _lib.check(e._handle, e.lib.vmb_track_update(e._handle, C.byref(a), _stream()), "vmb_track_update")


def _iterate_one(tr, live, gi):
    """The step of group gi alone on iteration 0's slice (the update is timed with the whole iteration)."""
    from vmap_b200 import _lib
    from vmap_b200.ensemble import _ptr
    a = _lib.TrackArgs()
    a.n_groups, a.n_iter, a.iter = len(live), tr.n_iter, 1
    a.pose, a.adam = _ptr(tr.pose), _ptr(tr.adam)
    a.colour_scaling, a.opacity_scaling = 5.0, 10.0
    for k, gr in enumerate(live):
        gr.bind(a.group[k], 0)
    _step(live[gi], a, gi, ba=False)


if __name__ == "__main__":
    main()
