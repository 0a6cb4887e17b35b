"""Timing of the 3-D metrics (vmap_b200.metrics): the exact nearest-neighbour kernel (vmb_nn_dist) at ref = query = 10 k
and 200 k surface samples of a trained sphere mesh and of a large marching-cubes mesh, with host cKDTree build + query
on the same points for comparison, and the whole calc_3d_metric for the object case (N = 10 k, crop to the GT box) and
the scene case (N = 200 k).  CUDA-event timings; the card and its power limit are read in the same run.  Writes one
JSON line.  Dev / profiling tool."""
import json, os, subprocess, sys, time, types
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from scipy.spatial import cKDTree
from oracle import vmap_oracle as vo
from vmap_b200 import mesh, metrics
from vmap_b200.ensemble import VmapEnsemble
from vmap_b200.lazy import bind_modules
from vmap_b200.trainer import Trainer

dev = torch.device("cuda:0")


def ev_time(fn, n=10, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def host_time(fn, n=3):
    fn()
    t0 = time.perf_counter()
    for _ in range(n): fn()
    return (time.perf_counter() - t0) / n * 1e3


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def trained_sphere_mesh():
    """Object 0 of a stack trained 150 steps on the analytic sphere scene, meshed at 128^3."""
    from oracle import scene
    from vmap_b200.utils import BoundingBox
    t = Trainer(types.SimpleNamespace(obj_id=1, training_device=dev, hidden_feature_size=32, obj_scale=2.0,
                                      n_unidir_funcs=5))
    ens = VmapEnsemble(2, hidden=32, scale=2.0)
    bind_modules(ens, 0, t.fc_occ_map, t.pe)
    ens.load_stacked(vo.init_params(2, 32, seed=3))
    for it in range(150):
        ens.step({k: v.to(dev) for k, v in scene.sphere_batch(2, 240, 10, seed=it).items()})
    b = BoundingBox()
    b.center, b.R, b.extent = np.zeros(3), np.eye(3), np.full(3, 1.2)
    return t.meshing(b, torch.zeros(3), grid_dim=128)


def mc_mesh(D, fn):
    x = torch.linspace(-1, 1, D, device=dev)
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    s = 2.0 / (D - 1)
    v, f, _ = mesh.marching_cubes(fn(X, Y, Z), 0.0, np.concatenate([np.eye(3) * s, np.full((3, 1), -1.0)], 1))
    return v, f


def uv_sphere(r, n_lat=200, n_lon=400):
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.concatenate([[[0, 0, r]], np.stack([r * np.sin(T) * np.cos(P), r * np.sin(T) * np.sin(P), r * np.cos(T)],
                                              -1).reshape(-1, 3), [[0, 0, -r]]])
    i = np.arange(n_lat - 2)[:, None]; j = np.arange(n_lon)[None, :]
    a, b = 1 + i * n_lon + j, 1 + i * n_lon + (j + 1) % n_lon
    c, d = a + n_lon, b + n_lon
    f = np.concatenate([np.stack([np.zeros(n_lon, int), 1 + np.arange(n_lon), 1 + (np.arange(n_lon) + 1) % n_lon], 1),
                        np.stack([a, c, d], -1).reshape(-1, 3), np.stack([a, d, b], -1).reshape(-1, 3),
                        np.stack([a[-1] + n_lon, np.full(n_lon, len(v) - 1), b[-1] + n_lon], 1)])
    return v, f


out = {"card": card()}
sphere = trained_sphere_mesh()
meshes = {"trained_sphere_128": (torch.from_numpy(np.asarray(sphere.vertices, np.float32)).to(dev),
                                 torch.from_numpy(np.asarray(sphere.faces, np.int32)).to(dev)),
          "mc_torus_384": mc_mesh(384, lambda X, Y, Z: 0.25 - torch.sqrt((torch.sqrt(X ** 2 + Y ** 2) - 0.55) ** 2 + Z ** 2))}
for name, m in meshes.items():
    for n in (10000, 200000):
        ref, _ = metrics.sample_surface(m, n, seed=0)
        qry, _ = metrics.sample_surface(m, n, seed=1)
        gpu_ms = ev_time(lambda: metrics.nn_dist(ref, qry))
        r64, q64 = ref.cpu().double().numpy(), qry.cpu().double().numpy()
        host_ms = host_time(lambda: cKDTree(r64).query(q64))
        d = metrics.nn_dist(ref, qry).cpu().double().numpy()
        err = float(np.abs(d - cKDTree(r64).query(q64)[0]).max())
        print(name, n, f"{gpu_ms:.3f} ms", f"{host_ms:.1f} ms", file=sys.stderr, flush=True)
        out[f"nn_{name}_{n // 1000}k"] = {"faces": int(m[1].shape[0]), "gpu_nn_ms": gpu_ms, "host_ckdtree_ms": host_ms,
                                          "max_abs_diff": err}

gt_obj = uv_sphere(0.45, 24, 48)                 # the GT box fit is a host convex hull over every hull face normal
out["gt_obj_vertices"] = int(len(gt_obj[0]))
out["host_gt_box_fit_ms"] = host_time(lambda: mesh.oriented_bounds(gt_obj[0]), n=2)
out["calc_3d_metric_obj_10k_crop_ms"] = ev_time(
    lambda: metrics.calc_3d_metric(sphere, gt_obj, N=10000, crop_to_gt_box=True), n=3, warm=1)
print("obj", out["calc_3d_metric_obj_10k_crop_ms"], file=sys.stderr, flush=True)
scene_rec = meshes["mc_torus_384"]
scene_gt = mc_mesh(384, lambda X, Y, Z: 0.26 - torch.sqrt((torch.sqrt(X ** 2 + Y ** 2) - 0.55) ** 2 + Z ** 2))
out["calc_3d_metric_scene_200k_ms"] = ev_time(lambda: metrics.calc_3d_metric(scene_rec, scene_gt, N=200000), n=5, warm=2)
out["scene_faces"] = [int(scene_rec[1].shape[0]), int(scene_gt[1].shape[0])]
print(json.dumps(out))
