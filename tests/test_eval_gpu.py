"""GPU: the 3-D metric kernels (K6: box crop, surface sampling, exact nearest neighbour) against oracle/eval_oracle.py
and scipy's cKDTree, vmap_b200.metrics on analytic meshes, and the evaluation of a trained two-object stack end to end
(meshing -> export -> load -> calc_3d_metric, and tools/eval_3d.py on a directory laid out like the reference's)."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import eval_oracle as eo
from oracle import scene
from oracle import vmap_oracle as vo
from tests._util import to_dev
from tests.test_eval_oracle import random_mesh, rot, uv_sphere

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- nearest neighbour ----------------------------------------------------------------------------------------------
def _nn_case(kind, n_ref, n_q, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        ref, q = rng.random((n_ref, 3)), rng.random((n_q, 3))
    elif kind == "blobs":                                        # tight blobs plus far outliers stretch the grid
        c = rng.normal(size=(5, 3))
        ref = c[rng.integers(0, 5, n_ref)] + rng.normal(size=(n_ref, 3)) * 1e-3
        ref[: max(1, n_ref // 100)] = rng.normal(size=(max(1, n_ref // 100), 3)) * 50
        q = c[rng.integers(0, 5, n_q)] + rng.normal(size=(n_q, 3)) * 3e-3
        q[: n_q // 10] = rng.normal(size=(n_q // 10, 3)) * 20
    elif kind == "outside":                                      # queries far outside ref's box
        ref = rng.random((n_ref, 3))
        q = rng.normal(size=(n_q, 3)) * 10
    elif kind == "duplicates":
        base = rng.random((n_ref // 4, 3))
        ref = base[rng.integers(0, len(base), n_ref)]
        q = rng.random((n_q, 3))
    else:                                                        # "flat": a planar ref set (zero-extent axis)
        ref = np.concatenate([rng.random((n_ref, 2)), np.zeros((n_ref, 1))], 1)
        q = rng.random((n_q, 3)) - 0.5
    return ref.astype(np.float32), q.astype(np.float32)


@pytest.mark.parametrize("kind,n_ref,n_q", [("uniform", 1, 100), ("uniform", 7, 1000), ("uniform", 1000, 1000),
                                            ("uniform", 200000, 200000), ("blobs", 20000, 20000),
                                            ("outside", 5000, 5000), ("duplicates", 4000, 4000), ("flat", 3000, 3000)])
def test_nn_dist_matches_kdtree(kind, n_ref, n_q):
    from vmap_b200.metrics import nn_dist
    ref, q = _nn_case(kind, n_ref, n_q, seed=n_ref + n_q)
    k = min(2, n_ref)
    d_ref, i_ref = cKDTree(ref.astype(np.float64)).query(q.astype(np.float64), k=k)
    d_ref, i_ref = d_ref.reshape(n_q, k), i_ref.reshape(n_q, k)
    d, idx = nn_dist(torch.from_numpy(ref).cuda(), torch.from_numpy(q).cuda(), with_index=True)
    d2, idx2 = nn_dist(torch.from_numpy(ref).cuda(), torch.from_numpy(q).cuda(), with_index=True)
    assert torch.equal(d, d2) and torch.equal(idx, idx2)                       # bitwise repeatable
    d, idx = d.cpu().numpy().astype(np.float64), idx.cpu().numpy()
    assert np.all(np.abs(d - d_ref[:, 0]) <= 1e-6 + 1e-6 * d_ref[:, 0])
    clear = d_ref[:, 1] > d_ref[:, 0] + 1e-5 if k == 2 else np.ones(n_q, bool)
    assert clear.mean() > (0.05 if kind == "duplicates" else 0.5)
    assert np.array_equal(idx[clear], i_ref[clear, 0])
    if kind == "duplicates":                                                   # ties go to the lowest index
        first = {}
        for j, p in enumerate(map(tuple, ref)):
            first.setdefault(p, j)
        assert all(first[tuple(ref[j])] == j for j in idx)


def test_nn_dist_bad_arguments():
    from vmap_b200 import _lib
    from vmap_b200.metrics import nn_dist
    with pytest.raises(_lib.VmbError):
        nn_dist(torch.zeros(0, 3, device="cuda"), torch.zeros(5, 3, device="cuda"))
    assert nn_dist(torch.zeros(3, 3, device="cuda"), torch.zeros(0, 3, device="cuda")).shape == (0,)


# ---- box crop -------------------------------------------------------------------------------------------------------
def _mc_sphere(D, r, device="cuda"):
    """Marching-cubes sphere of radius r on a D^3 grid over [-1, 1]^3 (vertices in world units)."""
    from vmap_b200.mesh import marching_cubes
    x = torch.linspace(-1, 1, D, device=device)
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    vol = r - torch.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    s = 2.0 / (D - 1)
    A = np.concatenate([np.eye(3) * s, np.full((3, 1), -1.0)], 1)
    v, f, _ = marching_cubes(vol, 0.0, A)
    return v, f


def _compare_clip(v, f, c, R, ext):
    from vmap_b200.metrics import crop_to_box
    v32 = np.asarray(v, np.float32)
    # the kernel takes the box in fp32: clip the oracle against the same box, since near-grazing edges move their
    # crossings by (plane error) / sin(angle)
    c, R, ext = (np.asarray(x, np.float32).astype(np.float64) for x in (c, R, ext))
    ref = eo.clip_to_box(v32, f, c, R, ext)
    out = crop_to_box((torch.from_numpy(v32).cuda(), torch.as_tensor(np.asarray(f)).cuda()), c, R, ext)
    if len(ref) == 0:
        assert out is None
        return ref
    out = out.cpu().numpy()
    assert out.shape == ref.shape
    assert np.abs(out - ref).max() < 1e-6
    return ref


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_clip_random_mesh_matches_oracle(seed):
    v, f = random_mesh(seed, nv=2000, nf=5000)
    ref = _compare_clip(v, f, np.array([0.05, -0.1, 0.0]), rot(seed + 20), np.array([0.7, 0.5, 0.9]))
    assert len(ref) > 500


def test_clip_mc_sphere_under_rotated_boxes():
    v, f = _mc_sphere(128, 0.6)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    for s in range(3):
        c = np.random.default_rng(s).normal(size=3) * 0.2
        ref = _compare_clip(v, f, c, rot(s + 30), np.array([0.8, 1.0, 0.6]))
        assert len(ref) > 1000


def test_clip_inside_all_and_outside_all():
    from vmap_b200 import _lib
    v, f = random_mesh(9)
    ref = _compare_clip(v, f, np.zeros(3), rot(1), np.full(3, 100.0))
    assert np.array_equal(ref, v.astype(np.float32)[f])
    assert len(_compare_clip(v, f, np.array([40.0, 0, 0]), rot(1), np.ones(3))) == 0
    # emit must follow a count of the same mesh and box
    from vmap_b200.mesh import _kernels, _p
    k = _kernels(torch.device("cuda:0"))
    vt, ft = torch.from_numpy(v.astype(np.float32)).cuda(), torch.from_numpy(f.astype(np.int32)).cuda()
    a = _lib.ClipArgs()
    a.vertices, a.n_vertices, a.faces, a.n_faces = _p(vt), len(v), _p(ft), len(f)
    a.rotation[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
    a.extent[:] = [1, 1, 1]
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    a.count = _p(cnt)
    k.call("vmb_clip_count", a)
    a.extent[0] = 2.0
    with pytest.raises(_lib.VmbError):
        k.call("vmb_clip_emit", a)


# ---- surface sampling -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["random", "mc_sphere"])
def test_sample_surface_injected_matches_oracle(which):
    from vmap_b200.metrics import sample_surface
    if which == "random":
        v, f = random_mesh(11, nv=500, nf=3000)
        v = v.astype(np.float32)
    else:
        vt, ft = _mc_sphere(96, 0.5)
        v, f = vt.cpu().numpy(), ft.cpu().numpy()
    N = 50000
    u = eo.uniforms(N, 12)
    p_ref, fi_ref = eo.sample_surface(v, f, u)
    p, fi = sample_surface((torch.from_numpy(v).cuda(), torch.as_tensor(f).cuda()), N, uniforms=u)
    assert np.array_equal(fi.cpu().numpy(), fi_ref)
    assert np.abs(p.cpu().numpy() - p_ref).max() < 1e-6


def test_sample_surface_philox_repeatable_and_seeded():
    from vmap_b200 import _lib
    from vmap_b200.metrics import sample_surface
    v, f = random_mesh(13)
    m = (v.astype(np.float32), f)
    a, fa = sample_surface(m, 20000, seed=5)
    b, fb = sample_surface(m, 20000, seed=5)
    c, _ = sample_surface(m, 20000, seed=6)
    assert torch.equal(a, b) and torch.equal(fa, fb)
    assert (a != c).any(dim=1).float().mean() > 0.99
    # area-proportional face counts from the Philox stream too
    from scipy.stats import chisquare
    area = eo.face_areas(v.astype(np.float32), f)
    obs = np.bincount(fa.cpu().numpy(), minlength=len(f))
    exp = 20000 * area / area.sum()
    keep = exp > 5
    assert chisquare(obs[keep], exp[keep] * obs[keep].sum() / exp[keep].sum()).pvalue > 1e-4
    with pytest.raises(_lib.VmbError):                                         # total area 0
        sample_surface((np.zeros((3, 3), np.float32), np.array([[0, 1, 2]])), 10)


# ---- metrics --------------------------------------------------------------------------------------------------------
def test_metrics_match_oracle():
    from vmap_b200 import metrics as M
    for name, n_gt, n_rec, kind, seed in eo.METRIC_CASES:
        gt, rec = eo.metric_points(n_gt, n_rec, kind, seed)
        gt, rec = gt.astype(np.float32), rec.astype(np.float32)
        # no gt -> rec distance within 1e-6 of a threshold, so fp32 rounding cannot flip a ratio
        d = cKDTree(rec.astype(np.float64)).query(gt.astype(np.float64))[0]
        gt = gt[(np.abs(d - 0.01) > 1e-6) & (np.abs(d - 0.05) > 1e-6)]
        for fn in ("accuracy", "completion", "chamfer"):
            assert getattr(M, fn)(gt, rec) == pytest.approx(getattr(eo, fn)(gt, rec), rel=1e-6, abs=1e-7), (name, fn)
        for th in (0.01, 0.05):
            assert M.completion_ratio(gt, rec, th) == eo.completion_ratio(gt, rec, th), (name, th)
        assert M.accuracy(torch.from_numpy(gt).cuda(), torch.from_numpy(rec).cuda()) == M.accuracy(gt, rec)


def test_concentric_spheres():
    from vmap_b200.metrics import calc_3d_metric
    rec, gt = _mc_sphere(256, 0.47), _mc_sphere(256, 0.45)
    m = calc_3d_metric(rec, gt, N=200000, seed=1)
    acc, comp, r1, r5 = (x[0] for x in m)
    print(f"concentric spheres: acc {acc:.5f} comp {comp:.5f} ratio@1cm {r1} ratio@5cm {r5}")
    assert acc == pytest.approx(0.02, abs=1e-3) and comp == pytest.approx(0.02, abs=1e-3)
    assert r1 < 1e-3 and r5 == 1.0


# ---- trained end to end ---------------------------------------------------------------------------------------------
R_SPHERE = 0.45                       # scene.sphere_batch: object 0 is a sphere of radius 0.45 at the origin


def _trainer(obj_id):
    from vmap_b200.trainer import Trainer
    return Trainer(types.SimpleNamespace(obj_id=obj_id, training_device="cuda:0", hidden_feature_size=32,
                                         obj_scale=2.0, n_unidir_funcs=5))


@pytest.fixture(scope="module")
def trained_mesh():
    """Object 0 of a two-object stack trained 500 steps on the analytic sphere scene, meshed at 64^3."""
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.lazy import bind_modules
    from vmap_b200.utils import BoundingBox
    trs = [_trainer(1), _trainer(2)]
    ens = VmapEnsemble(2, hidden=32, scale=2.0, impl="umma")
    for i, t in enumerate(trs):
        bind_modules(ens, i, t.fc_occ_map, t.pe)
    ens.load_stacked(vo.init_params(2, 32, seed=5))
    for it in range(500):
        ens.step(to_dev(scene.sphere_batch(2, 240, 10, seed=1000 + it)))
    ens.check_status()
    b = BoundingBox()
    b.center, b.R, b.extent = np.zeros(3), np.eye(3), np.full(3, 1.2)
    m = trs[0].meshing(b, torch.zeros(3), grid_dim=64)
    assert m is not None
    return m


def test_trained_mesh_metric_matches_oracle_pipeline(trained_mesh):
    from vmap_b200.metrics import calc_3d_metric
    gv, gf = uv_sphere(R_SPHERE, 60, 120)
    gv = gv.astype(np.float32)
    N = 10000
    u_rec, u_gt = eo.uniforms(N, 21), eo.uniforms(N, 22)
    rv = np.asarray(trained_mesh.vertices, np.float32)
    m = calc_3d_metric(trained_mesh, (gv, gf), N=N, crop_to_gt_box=True, uniforms=(u_rec, u_gt))
    ref = eo.calc_3d_metric(rv, trained_mesh.faces, gv, gf, u_rec, u_gt, crop_to_gt_box=True)
    print("trained sphere vs GT:", m, "oracle:", ref)
    assert np.allclose(np.array(m), np.array(ref), rtol=0, atol=1e-5)
    assert m[0][0] < 0.1 and m[1][0] < 0.02 and m[3][0] > 0.9   # the trained sphere is close to the GT sphere


def test_exported_mesh_scores_like_in_memory(trained_mesh, tmp_path):
    from vmap_b200.metrics import calc_3d_metric, load_mesh
    gt = uv_sphere(R_SPHERE, 60, 120)
    p = str(tmp_path / "frame_1999_obj1.obj")
    trained_mesh.export(p)
    a = calc_3d_metric(trained_mesh, gt, N=10000, crop_to_gt_box=True, seed=3)
    b = calc_3d_metric(load_mesh(p), gt, N=10000, crop_to_gt_box=True, seed=3)
    assert np.allclose(np.array(a), np.array(b), rtol=0, atol=1e-6)


def _write_ply(path, v, f):
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", "property float x",
            "property float y", "property float z", f"element face {len(f)}",
            "property list uchar int vertex_indices", "property int object_id", "end_header"]
    body = np.asarray(v, "<f4").tobytes()
    rec = np.zeros(len(f), np.dtype([("n", "u1"), ("i", "<i4", (3,)), ("o", "<i4")]))
    rec["n"], rec["i"] = 3, f
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode() + body + rec.tobytes())


def test_eval_3d_tool(trained_mesh, tmp_path):
    mesh_dir, gt_dir, out = tmp_path / "scene_mesh", tmp_path / "room_0" / "habitat", tmp_path / "eval_mesh"
    mesh_dir.mkdir(); gt_dir.mkdir(parents=True)
    trained_mesh.export(str(mesh_dir / "frame_1999_obj1.obj"))
    trained_mesh.export(str(mesh_dir / "frame_1999_obj0.obj"))
    gv, gf = uv_sphere(R_SPHERE, 40, 80)
    _write_ply(gt_dir / "mesh_semantic.ply_1.ply", gv, gf)                 # object 1 (class 7)
    _write_ply(gt_dir / "mesh_semantic.ply_3.ply", gv[gf[:len(gf) // 2]].reshape(-1, 3),
               np.arange(3 * (len(gf) // 2)).reshape(-1, 3))                 # background: two halves (classes 5, 12)
    _write_ply(gt_dir / "mesh_semantic.ply_4.ply", gv[gf[len(gf) // 2:]].reshape(-1, 3),
               np.arange(3 * (len(gf) - len(gf) // 2)).reshape(-1, 3))
    _write_ply(gt_dir.parent / "mesh.ply", gv, gf)
    (gt_dir / "info_semantic.json").write_text(json.dumps({"objects": [
        {"id": 1, "class_id": 7}, {"id": 3, "class_id": 5}, {"id": 4, "class_id": 12}]}))
    tool = os.path.join(ROOT, "tools", "eval_3d.py")
    for mode in ("obj", "scene"):
        r = subprocess.run([sys.executable, tool, "--mode", mode, "--mesh-dir", str(mesh_dir), "--gt-dir", str(gt_dir),
                            "--out", str(out)], capture_output=True, text=True, cwd=ROOT, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "Acc | Comp | Comp Ratio 1cm | Comp Ratio 5cm" in r.stdout
    assert np.load(out / "metric_obj1.npy").shape == (4, 1) and np.load(out / "metric_obj0.npy").shape == (4, 1)
    obj = np.load(out / "metrics_3D_obj.npy")
    assert obj.shape == (4, 2, 1)
    assert np.load(out / "metrics_3D_scene.npy").shape == (4, 1, 1)
    # the tool's numbers are calc_3d_metric's on the files it read (object 1: 10 000 samples, cropped)
    from vmap_b200.metrics import calc_3d_metric, load_mesh
    m1 = calc_3d_metric(load_mesh(str(mesh_dir / "frame_1999_obj1.obj")), load_mesh(str(gt_dir / "mesh_semantic.ply_1.ply")),
                        N=10000, crop_to_gt_box=True, seed=0)
    assert np.allclose(obj[:, 1], np.array(m1), rtol=0, atol=1e-9)
