"""Timing of the meshing block (train.py:343-368): sceneObject.get_bound (GPU unprojection + host hull / box fit) and
Trainer.meshing's stages (grid evaluation, marching cubes count + emit, vertex colours) at grid 128 and 256, for one
object of a 20-object hidden-32 stack and for a hidden-128 background model.  CUDA-event timings; the card and its
power limit are read in the same run.  Writes one JSON line.  Dev / profiling tool."""
import json, os, subprocess, sys, time, types
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from oracle import vmap_oracle as vo
from vmap_b200 import mesh
from vmap_b200.ensemble import VmapEnsemble
from vmap_b200.lazy import bind_modules
from vmap_b200.trainer import Trainer, make_3D_grid

dev = torch.device("cuda:0")


def ev_time(fn, n=5, warm=2):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def sphere_params(n_obj, hidden, seed):
    """A stack trained briefly on the analytic sphere scene, so that the meshes have realistic sizes."""
    from oracle import scene
    ens = VmapEnsemble(n_obj, hidden=hidden, scale=2.0)
    ens.load_stacked(vo.init_params(n_obj, hidden, seed=seed))
    for it in range(150):
        ens.step({k: v.to(dev) for k, v in scene.sphere_batch(n_obj, 240, 10, seed=it).items()})
    torch.cuda.synchronize()
    return ens


out = {"card": card()}
for name, n_obj, hidden in (("obj_of_20_h32", 20, 32), ("bg_h128", 1, 128)):
    ens = sphere_params(n_obj, hidden, seed=3)
    trained = ens.params.clone()
    t = Trainer(types.SimpleNamespace(obj_id=1, training_device=dev, hidden_feature_size=hidden, obj_scale=2.0,
                                      n_unidir_funcs=5))
    bind_modules(ens, 0, t.fc_occ_map, t.pe)         # binding copies the module's init into row 0: restore it
    ens.params.copy_(trained)
    ens.refresh_image()
    bound = types.SimpleNamespace(center=np.zeros(3), R=np.eye(3), extent=np.full(3, 1.2))
    for D in (128, 256):
        s = bound.extent / (2 * t.bound_extent)
        grid = make_3D_grid(dim=D, device=dev, scale=torch.from_numpy(s).float().to(dev)).view(-1, 3)
        occ = {}
        def grid_eval():
            occ["v"] = t.eval_points(grid)[0]
        A = np.concatenate([np.diag(s) * (2.0 / (D - 1)), -s[:, None]], 1)
        res = {}
        def mc():
            res["m"] = mesh.marching_cubes(occ["v"].view(D, D, D), 0.5, A)
        grid_ms = ev_time(grid_eval)
        mc_ms = ev_time(mc)                          # includes the one host sync between count and emit
        if res["m"] is None:
            out[f"{name}_D{D}"] = {"grid_eval_ms": grid_ms, "mc_count_emit_ms": mc_ms, "vertices": 0}
            continue
        verts = res["m"][0]
        col_ms = ev_time(lambda: t.eval_points(verts))
        t.meshing(bound, torch.zeros(3), grid_dim=D)
        t0 = time.perf_counter()
        for _ in range(3):
            t.meshing(bound, torch.zeros(3), grid_dim=D)
        torch.cuda.synchronize()
        out[f"{name}_D{D}"] = {"grid_eval_ms": grid_ms, "mc_count_emit_ms": mc_ms, "vertex_colour_ms": col_ms,
                               "meshing_total_ms": (time.perf_counter() - t0) / 3 * 1e3,
                               "vertices": int(verts.shape[0]), "faces": int(res["m"][1].shape[0])}

# get_bound: 20 keyframes of 1200 x 680, ~25 % of the pixels on the object
W, H, KF = 1200, 680, 20
g = torch.Generator().manual_seed(0)
rgbs = torch.zeros(KF + 1, W, H, 4, dtype=torch.uint8)
u = torch.arange(W)[:, None]; v = torch.arange(H)[None, :]
rgbs[:KF, :, :, 3] = (((u - 600) ** 2 / 300 ** 2 + (v - 340) ** 2 / 200 ** 2) < 1).to(torch.uint8)
depth = (torch.rand(KF + 1, W, H, generator=g) * 0.5 + 1.5)
twc = torch.eye(4).repeat(KF + 1, 1, 1)
for k in range(KF):
    a = 2 * np.pi * k / KF
    twc[k, :3, :3] = torch.tensor([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], dtype=torch.float32)
obj = types.SimpleNamespace(data_device=dev, frames_width=W, frames_height=H, n_keyframes=KF, obj_id=1, store=None,
                            rgbs_batch=rgbs.to(dev), depth_batch=depth.to(dev), t_wc_batch=twc.to(dev))
K = np.array([[600.0, 0, 599.5], [0, 600.0, 339.5], [0, 0, 1]])
pts = {}
def unproj():
    pts["p"] = mesh.unproject_object(obj, K)
unproj_ms = ev_time(unproj)
p = pts["p"].cpu().numpy()
t0 = time.perf_counter()
mesh.oriented_bounds(p)
out["get_bound"] = {"points": int(p.shape[0]), "gpu_unproject_ms": unproj_ms,
                    "host_hull_box_ms": (time.perf_counter() - t0) * 1e3}
print(json.dumps(out))
