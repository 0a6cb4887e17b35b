"""Timing of the device convex hull + minimum-volume box (K8, mesh.oriented_bounds_gpu) against scipy's qhull + the
host fit (mesh.oriented_bounds) on: the 3.8 M-point get_bound scene of tools/mesh_time.py, the 1.1 k-vertex GT of the
per-object metric (UV sphere), a noisy sphere shell and the all-extreme worst case (integer paraboloid).  Host clock
around calls that end in a device sync (the box download); median and spread over repeats; the card and its power
limit are read in the same run.  Writes one JSON line.  Dev / profiling tool."""
import json, os, subprocess, sys, time, types
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from vmap_b200 import mesh

dev = torch.device("cuda:0")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def wall(fn, n, warm):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": float(np.median(ts)), "min_ms": float(np.min(ts)), "max_ms": float(np.max(ts))}


def get_bound_points():
    W, H, KF = 1200, 680, 20                       # tools/mesh_time.py's scene
    g = torch.Generator().manual_seed(0)
    rgbs = torch.zeros(KF + 1, W, H, 4, dtype=torch.uint8)
    u = torch.arange(W)[:, None]; v = torch.arange(H)[None, :]
    rgbs[:KF, :, :, 3] = (((u - 600) ** 2 / 300 ** 2 + (v - 340) ** 2 / 200 ** 2) < 1).to(torch.uint8)
    depth = (torch.rand(KF + 1, W, H, generator=g) * 0.5 + 1.5)
    twc = torch.eye(4).repeat(KF + 1, 1, 1)
    for k in range(KF):
        a = 2 * np.pi * k / KF
        twc[k, :3, :3] = torch.tensor([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]],
                                      dtype=torch.float32)
    obj = types.SimpleNamespace(data_device=dev, frames_width=W, frames_height=H, n_keyframes=KF, obj_id=1, store=None,
                                rgbs_batch=rgbs.to(dev), depth_batch=depth.to(dev), t_wc_batch=twc.to(dev))
    K = np.array([[600.0, 0, 599.5], [0, 600.0, 339.5], [0, 0, 1]])
    return mesh.unproject_object(obj, K)


def uv_sphere(r, n_lat, n_lon):
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    t, p = np.meshgrid(th, ph, indexing="ij")
    ring = np.stack([np.sin(t) * np.cos(p), np.sin(t) * np.sin(p), np.cos(t)], -1).reshape(-1, 3)
    return r * np.concatenate([[[0, 0, 1.0]], ring, [[0, 0, -1.0]]])


rng = np.random.default_rng(0)
x = rng.normal(size=(200000, 3))
g = np.arange(-50, 50, dtype=np.float64)
gx, gy = [a.ravel() for a in np.meshgrid(g, g, indexing="ij")]
cases = {
    "get_bound_scene": get_bound_points(),
    "gt_uv_sphere": torch.from_numpy(uv_sphere(0.45, 30, 38)).to(dev),
    "shell_200k": torch.from_numpy(x / np.linalg.norm(x, axis=1, keepdims=True)
                                   * (1 + 1e-3 * rng.normal(size=(200000, 1)))).to(dev),
    "paraboloid_all_extreme_10k": torch.from_numpy(np.column_stack([gx, gy, gx * gx + gy * gy])).to(dev),
}
out = {"card": card()}
for name, pts in cases.items():
    host = pts.double().cpu().numpy()
    hull = mesh.convex_hull(pts)
    r = {"points": int(pts.shape[0]), "hull_vertices": int(hull.vertices.numel())}
    r["gpu_hull_ms"] = wall(lambda: mesh.convex_hull(pts), n=5, warm=1)
    r["gpu_hull_box_ms"] = wall(lambda: mesh.oriented_bounds_gpu(pts), n=5, warm=1)
    _, _, e_gpu = mesh.oriented_bounds_gpu(pts)
    if name != "paraboloid_all_extreme_10k":        # qhull + the host fit over 10 k facet normals takes minutes
        t0 = time.perf_counter()
        _, _, e_host = mesh.oriented_bounds(host)
        r["host_qhull_box_ms"] = (time.perf_counter() - t0) * 1e3
        r["volume_rel_diff"] = float(abs(np.prod(e_gpu) / np.prod(e_host) - 1))
    out[name] = r
print(json.dumps(out))
