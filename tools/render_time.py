"""Timing of render_view (vmap_b200/render.py): a 1200 x 680 view of 20 hidden-32 objects trained 150 steps on the
sphere scene and placed on a 5 x 4 grid, plus a hidden-128 background source whose box spans the layout, at the
default sample counts.  Per-stage CUDA-event times (count, emit, forward, composite of each pass, summed over the ray
chunks), the whole call (median of 5), the points evaluated, and the card and its power limit read in the same run.
Writes one JSON line.  Dev / profiling tool."""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from oracle import scene
from oracle import vmap_oracle as vo
from vmap_b200 import render
from vmap_b200.ensemble import VmapEnsemble

dev = torch.device("cuda:0")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def trained(n_obj, hidden, seed):
    ens = VmapEnsemble(n_obj, hidden=hidden, scale=2.0)
    ens.load_stacked(vo.init_params(n_obj, hidden, seed=seed))
    for it in range(150):
        ens.step({k: v.to(dev) for k, v in scene.sphere_batch(n_obj, 240, 10, seed=it).items()})
    torch.cuda.synchronize()
    return ens


objs, bg = trained(20, 32, 3), trained(1, 128, 4)
srcs = []
for i in range(20):
    c = np.array([(i % 5 - 2) * 1.2, (i // 5 - 1.5) * 1.2, 4.0 + 0.3 * (i % 3)])
    srcs.append(render.Source(objs, i, i + 1, c, np.eye(3), np.full(3, 0.7), c))
srcs.append(render.Source(bg, 0, 0, np.array([0.0, 0.0, 4.3]), np.eye(3), np.array([3.4, 2.6, 1.2]),
                          np.array([0.0, 0.0, 4.3])))
W, H = 1200, 680
K = np.array([[600.0, 0, 599.5], [0, 600.0, 339.5], [0, 0, 1]])
T = np.eye(4)
kw = dict(near=0.0, far=10.0)
img, stats = render.render_view(srcs, T, K, W, H, **kw)        # warm-up
torch.cuda.synchronize()
stages = {}
render.render_view(srcs, T, K, W, H, stages=stages, **kw)
torch.cuda.synchronize()
stage_ms = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in stages.items()}
times = []
for _ in range(5):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    render.render_view(srcs, T, K, W, H, **kw)
    torch.cuda.synchronize()
    times.append((time.perf_counter() - t0) * 1e3)
print(json.dumps({"card": card(), "view": [W, H], "sources": len(srcs), "stage_ms": stage_ms,
                  "render_view_ms_median": float(np.median(times)), "points_coarse": stats["points_coarse"],
                  "points_fine": stats["points_fine"], "overflow_rays": stats["overflow_rays"],
                  "covered_pixels": int((img["instance"] >= 0).sum())}))
