"""GPU: the marching-cubes and unprojection kernels (K5) against oracle/mesh_oracle.py, and the meshing block of
train.py (get_bound -> meshing -> export, train.py:343-360) on a trained two-object stack."""
import types

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from oracle import scene
from oracle import vmap_oracle as vo
from tests._util import to_dev

pytestmark = pytest.mark.gpu


def _sphere(n, r=0.7):
    x = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    return (1.0 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2) / r).astype(np.float32)


def _torus(n):
    x = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    return (0.25 - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.55) ** 2 + Z ** 2)).astype(np.float32)


def _compare(vol, level, affine=None, vtol=1e-5):
    from vmap_b200.mesh import marching_cubes
    ov, of, on = mo.marching_cubes(vol, level, affine)
    out = marching_cubes(torch.from_numpy(vol).cuda(), level, affine)
    assert out is not None
    gv, gf, gn = (t.cpu().numpy() for t in out)
    assert gf.shape == of.shape and np.array_equal(gf, of)
    assert np.abs(gv - ov).max() < vtol
    assert np.abs(gn - on).max() < 1e-4
    return gv, gf


@pytest.mark.parametrize("shape,seed", [((17, 19, 23), 0), ((17, 19, 23), 1), ((31, 8, 5), 2), ((2, 3, 2), 3)])
def test_mc_random_volume_matches_oracle(shape, seed):
    vol = np.random.default_rng(seed).random(shape).astype(np.float32)
    _compare(vol, 0.5)


@pytest.mark.parametrize("n,fn", [(64, _sphere), (64, _torus), (256, _sphere), (256, _torus)])
def test_mc_analytic_volume_matches_oracle(n, fn):
    v, f = _compare(fn(n), 0.0)
    assert mo.directed_edge_check(f)


def test_mc_affine_matches_oracle():
    rng = np.random.default_rng(4)
    Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    A = np.concatenate([Q @ np.diag([0.02, 0.03, 0.025]), [[0.3], [-1.0], [2.0]]], 1)
    _compare(_sphere(48), 0.0, A, vtol=1e-5)


def test_mc_empty_volumes_and_bad_arguments():
    import ctypes as C
    from vmap_b200 import _lib
    from vmap_b200.mesh import _kernels, marching_cubes
    for v in (torch.zeros(9, 10, 11, device="cuda"), torch.ones(9, 10, 11, device="cuda")):
        assert marching_cubes(v, 0.5) is None
    k = _kernels(torch.device("cuda:0"))
    a = _lib.McArgs()
    vol = torch.zeros(1, 4, 4, device="cuda")          # nx < 2
    totals = torch.zeros(2, dtype=torch.int32, device="cuda")
    a.volume, a.nx, a.ny, a.nz, a.totals = C.c_void_p(vol.data_ptr()), 1, 4, 4, C.c_void_p(totals.data_ptr())
    a.affine[:] = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]
    with pytest.raises(_lib.VmbError):
        k.call("vmb_mc_count", a)
    vol2 = torch.zeros(3, 4, 4, device="cuda")
    a.volume, a.nx, a.affine[0] = C.c_void_p(vol2.data_ptr()), 3, 0.0
    with pytest.raises(_lib.VmbError):                 # singular affine
        k.call("vmb_mc_count", a)
    a.affine[0] = 1.0
    k.call("vmb_mc_count", a)
    assert totals.tolist() == [0, 0]
    a.nz = 5                                           # emit must follow a count of the same volume
    with pytest.raises(_lib.VmbError):
        k.call("vmb_mc_emit", a)


# ---- unprojection ---------------------------------------------------------------------------------------------------
def _frames(W, H, KF, seed):
    g = torch.Generator().manual_seed(seed)
    depth = torch.rand(KF, W, H, generator=g) * 3 + 0.5
    depth[torch.rand(KF, W, H, generator=g) < 0.2] = 0
    inst = (torch.rand(KF, W, H, generator=g) * 5).long().to(torch.int32)          # 0..4, obj 3 ~ 20 %
    inst[torch.rand(KF, W, H, generator=g) < 0.05] = -1
    twc = torch.eye(4).repeat(KF, 1, 1)
    for k in range(KF):
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g))
        twc[k, :3, :3] = q * torch.sign(torch.det(q))
        twc[k, :3, 3] = torch.randn(3, generator=g)
    rgb = torch.randint(0, 256, (KF, W, H, 3), generator=g).to(torch.uint8)
    return rgb, depth, inst, twc


@pytest.mark.parametrize("layout", ["per_object", "store"])
def test_unproject_matches_oracle(layout):
    from vmap_b200.keyframes import FrameStore
    from vmap_b200.mesh import unproject_object
    W, H, KF, n_kf, oid = 40, 30, 6, 4, 3
    rgb, depth, inst, twc = _frames(W, H, KF, seed=7)
    K = np.array([[35.0, 0, 19.5], [0, 33.0, 14.5], [0, 0, 1]])
    o = types.SimpleNamespace(data_device="cuda:0", frames_width=W, frames_height=H, n_keyframes=n_kf, obj_id=oid)
    if layout == "store":
        st = FrameStore(W, H, 8, "cuda:0")
        slots = [st.put(rgb[k].cuda(), depth[k].cuda(), inst[k].cuda(), twc[k].cuda()) for k in range(KF)]
        o.store, o.kf_store_slot = st, slots[::-1]                    # keyframe k lives in slot KF-1-k
        order = list(range(KF))[::-1][:n_kf]
        ref = mo.unproject(depth.numpy()[order], (inst.numpy() == oid)[order], twc.numpy()[order], 35.0, 33.0, 19.5, 14.5)
    else:
        state = torch.where(inst == oid, 1, torch.where(inst == -1, 2, 0)).to(torch.uint8)
        o.store = None
        o.rgbs_batch = torch.cat([rgb, state[..., None]], -1).contiguous().cuda()
        o.depth_batch, o.t_wc_batch = depth.cuda(), twc.cuda()
        ref = mo.unproject(depth.numpy()[:n_kf], (inst.numpy() == oid)[:n_kf], twc.numpy()[:n_kf], 35.0, 33.0, 19.5, 14.5)
    pts = unproject_object(o, K).cpu().numpy()
    assert pts.shape == ref.shape and len(ref) > 500
    # same (keyframe, u, v) order, fp32 arithmetic
    assert np.allclose(pts, ref, rtol=1e-5, atol=1e-5)
    o.n_keyframes = 0
    assert unproject_object(o, K).shape == (0, 3)


# ---- trained end to end ---------------------------------------------------------------------------------------------
R_SPHERE = 0.45                       # scene.sphere_batch: object 0 is a sphere of radius 0.45 at the origin


def _trainer(obj_id):
    from vmap_b200.trainer import Trainer
    return Trainer(types.SimpleNamespace(obj_id=obj_id, training_device="cuda:0", hidden_feature_size=32,
                                         obj_scale=2.0, n_unidir_funcs=5))


@pytest.fixture(scope="module")
def trained():
    """Two objects trained 500 steps on the analytic sphere scene with the fused tensor-core step (bitwise
    reproducible); the Trainers' modules are views of the packed rows, as after update_vmap."""
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.lazy import bind_modules
    trs = [_trainer(1), _trainer(2)]
    ens = VmapEnsemble(2, hidden=32, scale=2.0, impl="umma")
    for i, t in enumerate(trs):
        bind_modules(ens, i, t.fc_occ_map, t.pe)
    ens.load_stacked(vo.init_params(2, 32, seed=5))
    for it in range(500):
        ens.step(to_dev(scene.sphere_batch(2, 240, 10, seed=1000 + it)))
    ens.check_status()
    return ens, trs


def _bound(extent=1.2):
    from vmap_b200.utils import BoundingBox
    b = BoundingBox()
    b.center, b.R, b.extent = np.zeros(3), np.eye(3), np.full(3, extent)
    return b


def _oracle_mesh(ens, row, trainer, bound, D):
    """CPU pipeline: oracle forward on the same grid -> oracle MC -> oracle colours."""
    from vmap_b200.trainer import make_3D_grid
    p = {k: v[row:row + 1].detach().cpu().clone() for k, v in ens.stacked().items()}
    sc = torch.tensor([2.0])
    s = np.asarray(bound.extent) / (2 * trainer.bound_extent)
    T = torch.eye(4)
    T[:3, :3] = torch.from_numpy(np.asarray(bound.R, np.float32))
    T[:3, 3] = torch.from_numpy(np.asarray(bound.center, np.float32))
    grid = make_3D_grid(dim=D, device="cuda:0", scale=torch.from_numpy(s).float().cuda(), transform=T.cuda()).view(-1, 3).cpu()
    with torch.no_grad():
        alpha, _ = vo.forward(p, sc, grid[None, :, None, :])
    occ = torch.sigmoid(alpha.view(D, D, D)).numpy()
    R, c = np.asarray(bound.R, np.float64), np.asarray(bound.center, np.float64)
    A = np.concatenate([R @ np.diag(s) * (2.0 / (D - 1)), (c - R @ s)[:, None]], 1)
    v, f, n = mo.marching_cubes(occ, 0.5, A)
    with torch.no_grad():
        _, col = vo.forward(p, sc, torch.from_numpy(v)[None, :, None, :])
    rgb = (col.view(-1, 3) * 255).to(torch.uint8).numpy()
    return occ, v, f, rgb, 2 * s.min() / (D - 1)


def test_trained_mesh_matches_cpu_pipeline(trained):
    from scipy.spatial import cKDTree
    ens, trs = trained
    D, bound = 64, _bound()
    occ_o, v_o, f_o, rgb_o, voxel = _oracle_mesh(ens, 0, trs[0], bound, D)
    assert mo.directed_edge_check(f_o) and len(f_o) > 1000
    r_o = np.linalg.norm(v_o, axis=1).mean()
    err_o = abs(r_o - R_SPHERE)
    print(f"oracle mesh: {len(v_o)} vertices, mean radius {r_o:.4f} (sphere {R_SPHERE}), voxel {voxel:.4f}")
    assert err_o < 0.15 * R_SPHERE, "training did not converge enough for the comparison to mean anything"
    # fp32 CUDA-core forward: the same mesh
    ens.impl = "fp32"
    m = trs[0].meshing(bound, torch.zeros(3), grid_dim=D)
    assert m is not None
    assert np.array_equal(m.faces, f_o)
    assert np.abs(m.vertices - v_o).max() < 1e-4
    assert np.abs(m.visual.vertex_colors[:, :3].astype(int) - rgb_o).max() <= 1
    assert (m.visual.vertex_colors[:, 3] == 255).all()
    assert np.allclose(np.linalg.norm(m.vertex_normals, axis=1), 1, atol=1e-5)
    # tensor-core forward (fp16 operands): close to it
    ens.impl = "umma"
    mt = trs[0].meshing(bound, torch.zeros(3), grid_dim=D)
    d1, _ = cKDTree(v_o).query(mt.vertices)
    d2, _ = cKDTree(mt.vertices).query(v_o)
    chamfer = 0.5 * (d1.mean() + d2.mean())
    r_t = np.linalg.norm(mt.vertices, axis=1).mean()
    print(f"tensor-core mesh: {len(mt.vertices)} vertices, chamfer {chamfer:.5f}, mean radius {r_t:.4f}")
    assert chamfer < 0.5 * voxel
    for mm in (m, mt):
        assert mo.directed_edge_check(mm.faces)
    assert abs(r_t - R_SPHERE) < err_o + 0.5 * voxel


def test_meshing_returns_none_without_a_surface(trained):
    ens, trs = trained
    t = _trainer(1)                                     # a private one-object ensemble
    with torch.no_grad():
        t.fc_occ_map.out_alpha.bias.fill_(-1e4)         # occupancy exactly 0 everywhere: "no occ"
    assert t.meshing(_bound(), torch.zeros(3), grid_dim=16) is None
    t2 = _trainer(2)
    with torch.no_grad():
        t2.fc_occ_map.out_alpha.weight.zero_()
        t2.fc_occ_map.out_alpha.bias.fill_(1.0)         # occupancy sigmoid(10) everywhere: no crossing
    assert t2.meshing(_bound(), torch.zeros(3), grid_dim=16) is None


def _render_keyframes(W, H, fx, n_views, seed):
    """Depth / instance images of the sphere (id 1, radius R_SPHERE at the origin) from cameras on a shell of radius
    2 looking at the origin, as sceneObject stores them ([W, H], u along W)."""
    g = torch.Generator().manual_seed(seed)
    cx, cy = (W - 1) / 2, (H - 1) / 2
    out = []
    for _ in range(n_views):
        o = torch.randn(3, generator=g, dtype=torch.float64)
        o = 2.0 * o / o.norm()
        z = -o / o.norm()
        x = torch.linalg.cross(z, torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64))
        x = x / x.norm()
        y = torch.linalg.cross(z, x)
        Rwc = torch.stack([x, y, z], 1)
        u = torch.arange(W, dtype=torch.float64)[:, None].expand(W, H)
        v = torch.arange(H, dtype=torch.float64)[None, :].expand(W, H)
        dc = torch.stack([(u - cx) / fx, (v - cy) / fx, torch.ones_like(u)], -1)     # z = 1: t is the z-depth
        dw = dc @ Rwc.T
        b = (dw * o).sum(-1)
        a = (dw * dw).sum(-1)
        c = (o * o).sum() - R_SPHERE ** 2
        disc = b * b - a * c
        hit = disc > 0
        t = (-b - torch.sqrt(disc.clamp_min(0))) / a
        depth = torch.where(hit, t, torch.full_like(t, 3.5)).float()
        inst = hit.to(torch.int32)
        twc = torch.eye(4)
        twc[:3, :3], twc[:3, 3] = Rwc.float(), o.float()
        rgb = torch.randint(0, 256, (W, H, 3), generator=g).to(torch.uint8)
        out.append((rgb, depth, inst, twc))
    return out, np.array([[fx, 0, cx], [0, fx, cy], [0, 0, 1.0]])


@pytest.mark.parametrize("layout", ["per_object", "store"])
def test_dropin_vis_block(trained, layout, tmp_path):
    """train.py:343-360 against the mirror API: get_bound, adaptive_grid_dim, meshing, export, read back."""
    import os
    from tests.test_mesh_oracle import read_obj
    from vmap_b200 import cfg as cfg_mod
    from vmap_b200.keyframes import FrameStore
    from vmap_b200.vmap import sceneObject
    ens, trs = trained
    d = cfg_mod.replica_room0_dict()
    W, H = 96, 64
    d["camera"].update(w=W, h=H, fx=60.0, fy=60.0, cx=(W - 1) / 2, cy=(H - 1) / 2)
    d["model"]["keyframe_buffer_size"] = 8
    d["model"]["keyframe_step"] = 1
    d["model"]["obj_scale"] = 2.0
    d["model"]["hidden_feature_size"] = 32
    d["trainer"]["do_bg"] = 0
    cfg = cfg_mod.Config(config_dict=d)
    frames, K = _render_keyframes(W, H, 60.0, 7, seed=3)
    store = FrameStore(W, H, 8, "cuda:0") if layout == "store" else None
    obj = None
    for fid, (rgb, depth, inst, twc) in enumerate(frames):
        bbox = torch.tensor([0.0, W - 1.0, 0.0, H - 1.0], device="cuda")
        if store is not None:
            slot = store.put(rgb.cuda(), depth.cuda(), inst.cuda(), twc.cuda(), frame_id=fid)
            args = (None, None, None, bbox, twc.cuda())
            if obj is None:
                obj = sceneObject(cfg, 1, *args, fid, store=store, frame_slot=slot)
            else:
                obj.append_keyframe(*args, frame_id=fid, frame_slot=slot)
            store.release(slot)
        else:
            state = inst.to(torch.uint8).cuda()
            args = (rgb.cuda(), depth.cuda(), state, bbox, twc.cuda())
            if obj is None:
                obj = sceneObject(cfg, 1, *args, fid)
            else:
                obj.append_keyframe(*args, frame_id=fid)
    assert obj.n_keyframes == 7
    # the trained object-0 network of the stack
    with torch.no_grad():
        for k, p in obj.trainer.fc_occ_map.named_parameters():
            p.copy_(dict(trs[0].fc_occ_map.named_parameters())[k])
        obj.trainer.pe.B_layer.weight.copy_(trs[0].pe.B_layer.weight)
    bound = obj.get_bound(K)                                                           # train.py:347
    assert bound is not None and obj.bbox3d is not None
    assert abs(np.linalg.det(bound.R) - 1) < 1e-6
    assert np.abs(np.asarray(bound.center)).max() < 0.05
    assert np.allclose(np.sort(bound.extent), 2 * R_SPHERE, atol=0.08)
    adaptive_grid_dim = int(np.minimum(np.max(bound.extent) // cfg.live_voxel_size + 1, cfg.grid_dim))   # train.py:351
    mesh = obj.trainer.meshing(bound, obj.obj_center, grid_dim=adaptive_grid_dim)                        # train.py:352
    assert mesh is not None
    out_dir = os.path.join(str(tmp_path), "scene_mesh")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "frame_{}_obj{}.obj".format(5, str(1)))                               # train.py:360
    mesh.export(path)
    v, c, n, f = read_obj(path)
    assert np.allclose(v, mesh.vertices, atol=1e-6) and np.array_equal(f, mesh.faces)
    assert np.array_equal(np.rint(c * 255).astype(np.uint8), mesh.visual.vertex_colors[:, :3])
    assert abs(np.linalg.norm(mesh.vertices, axis=1).mean() - R_SPHERE) < 0.05
    obj.save_checkpoints(str(tmp_path), 5)                                                                # train.py:385
    ck = torch.load(os.path.join(str(tmp_path), "obj_1_frame_5.pth"), weights_only=False)
    assert np.allclose(ck["bbox"].extent, bound.extent)
