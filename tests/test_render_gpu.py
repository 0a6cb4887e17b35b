"""GPU tests of the view renderer (K9, vmap_b200/render.py) against the numpy oracle (oracle/render_oracle.py):
bitwise geometry, full views on the fp32 and tensor-core forwards, chunking / reproducibility, empty cases, argument
checks, and trained quality on an analytic multi-sphere scene."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import render_oracle as ro
from oracle import scene
from oracle import vmap_oracle as vo
from vmap_b200 import _lib, render
from vmap_b200.ensemble import VmapEnsemble, _ptr

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
K48 = np.array([[40.0, 0, 23.5], [0, 40.0, 17.5], [0, 0, 1]])


def rot(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def random_scene(seed, n_src=6, edge=False):
    """Camera at the origin looking down +z; boxes in front, plus (edge) one containing the camera, one behind it,
    one off-screen, and 18 thin boxes stacked on the central ray (overflow)."""
    rng = np.random.default_rng(seed)
    T = np.eye(4)
    T[:3, :3] = rot(seed + 50) if seed % 2 else np.eye(3)
    T[:3, 3] = rng.normal(size=3) * 0.2
    boxes = []
    for i in range(n_src):
        c = T[:3, :3] @ (rng.normal([0, 0, 2.5], [0.5, 0.4, 0.6])) + T[:3, 3]
        boxes.append((c, rot(seed * 31 + i), rng.uniform(0.15, 0.6, 3)))
    if edge:
        boxes.append((T[:3, 3] + 0.05, np.eye(3), np.array([0.3, 0.3, 0.3])))          # camera inside
        boxes.append((T[:3, 3] - 3 * T[:3, 2], np.eye(3), np.array([0.5, 0.5, 0.5])))  # behind
        boxes.append((T[:3, 3] + 2 * T[:3, 2] + 9 * T[:3, 0], np.eye(3), np.full(3, 0.3)))   # off-screen
        for j in range(18):
            boxes.append((T[:3, 3] + (1.0 + 0.2 * j) * T[:3, 2], T[:3, :3], np.array([0.05, 0.05, 0.05])))
        boxes.append((np.array([0.3, 0.0, 2.0]) + T[:3, 3], np.eye(3), np.array([0.3, 0.2, 0.25])))  # face-aligned
    return T, boxes


def make_sources(boxes, ens_list):
    """Source i uses row i % n of ensemble (i % len(ens_list))."""
    out = []
    for i, (c, R, h) in enumerate(boxes):
        e = ens_list[i % len(ens_list)]
        out.append(render.Source(e, (i // len(ens_list)) % e.n_obj, 10 + i, c, R, h))
    return out


def nets_of(sources):
    cache = {}
    def net(s, pts):
        src = sources[s]
        key = (id(src.ens), src.row)
        if key not in cache:
            p = {k: v[src.row:src.row + 1].detach().cpu() for k, v in src.ens.stacked().items()}
            cache[key] = ro.oracle_net(p, float(src.ens.scale[src.row]))
        return cache[key](pts)
    return net


CENTRES = np.array([[-0.5, 0.0, 0.0], [0.3, 0.1, 0.6], [0.9, -0.2, 1.2], [-0.2, 0.5, 1.8]])


def trained_ens(n_obj, hidden, steps=150, seed=0, centres=None):
    """A stack trained on the sphere scene; with ``centres`` object i's sphere sits at centres[i] in world
    coordinates (sphere_batch's points shifted per object), as real objects are trained."""
    ens = VmapEnsemble(n_obj, hidden=hidden, scale=2.0)
    ens.load_stacked(vo.init_params(n_obj, hidden, seed=seed))
    shift = None if centres is None else torch.as_tensor(centres[:n_obj], dtype=torch.float32).view(n_obj, 1, 1, 3)
    for it in range(steps):
        b = scene.sphere_batch(n_obj, 240, 10, seed=it)
        if shift is not None:
            b["pcs"] = (b["pcs"] + shift).contiguous()
        ens.step({k: v.to(dev) for k, v in b.items()})
    torch.cuda.synchronize()
    return ens


@pytest.fixture(scope="module")
def ens32():
    return trained_ens(4, 32, seed=1, centres=CENTRES)


@pytest.fixture(scope="module")
def ens128():
    return trained_ens(1, 128, seed=2)


def gpu_pass(sources, T, K, W, H, n_coarse, n_fine, eps, near, far, p, zstar=None, state=None):
    """Run count + emit of pass p over the whole view in one chunk; returns the device tables."""
    v = render._View(sources, T, K, W, H, n_coarse, n_fine, eps, near, far)
    a, n = v.a, W * H
    st = state if state is not None else {
        "hit_src": torch.empty(n, 16, dtype=torch.int32, device=dev),
        "hit_t": torch.empty(n, 16, 2, dtype=torch.float64, device=dev),
        "hit_count": torch.empty(n, dtype=torch.int32, device=dev),
        "small": torch.zeros(1 + len(sources), dtype=torch.int32, device=dev)}
    a.hit_src, a.hit_t, a.hit_count = _ptr(st["hit_src"]), _ptr(st["hit_t"]), _ptr(st["hit_count"])
    a.overflow, a.src_total = _ptr(st["small"]), C.c_void_p(st["small"].data_ptr() + 4)
    st["zstar"] = zstar
    a.zstar = _ptr(zstar)
    a.ray0, a.n_rays = 0, n
    setattr(a, "pass", p)
    v.call("vmb_render_count", "count")
    small = st["small"].cpu()
    tot = small[1:].numpy().astype(np.int64)
    N = max(int(tot.sum()), 1)
    pts = torch.empty(N, 3, device=dev)
    z = torch.empty(N, device=dev)
    base = torch.empty(n, 16, dtype=torch.int32, device=dev)
    a.points, a.z, a.base = _ptr(pts), _ptr(z), _ptr(base)
    v.call("vmb_render_emit", "emit")
    torch.cuda.synchronize()
    return st, {"overflow": int(small[0]), "totals": tot, "points": pts[:int(tot.sum())].cpu().numpy(),
                "z": z[:int(tot.sum())].cpu().numpy(), "base": base.cpu().numpy()}


@pytest.mark.parametrize("seed,edge,near", [(0, False, 0.05), (1, True, 0.05), (2, True, 0.0), (3, False, 0.0)])
def test_geometry_bitwise(ens32, seed, edge, near):
    W, H, nc, nf, eps, far = 48, 36, 8, 4, 0.1, 6.0
    T, boxes = random_scene(seed, edge=edge)
    srcs = make_sources(boxes, [ens32])
    bt = render.box_table(srcs)
    o, d = ro.rays(W, H, K48, T)
    src, ht, cnt, ovf = ro.hit_table(bt, o, d, near, far)
    zbuf = torch.full((W * H,), -1.0, device=dev)
    st, g = gpu_pass(srcs, T, K48, W, H, nc, nf, eps, near, far, 0, zstar=zbuf)
    assert np.array_equal(st["hit_count"].cpu().numpy(), cnt)
    assert np.array_equal(st["hit_src"].cpu().numpy(), src)
    assert np.array_equal(st["hit_t"].cpu().numpy().view(np.int64), ht.view(np.int64))
    assert g["overflow"] == ovf and (ovf > 0) == edge
    c = ro.samples(bt, o, d, src, ht, cnt, nc)
    assert np.array_equal(g["totals"], c["totals"])
    assert np.array_equal(g["points"].view(np.int32), c["points"].view(np.int32))
    assert np.array_equal(g["z"].view(np.int32), c["z"].view(np.int32))
    used = c["counts"] > 0
    assert np.array_equal(g["base"][used], c["base"][used])
    # pass 1 with an injected z*: the oracle's fine positions, bitwise
    rng = np.random.default_rng(seed)
    zs = np.where(rng.random(W * H) < 0.7, rng.uniform(0.5, 4.0, W * H), -1.0).astype(np.float32)
    zbuf.copy_(torch.from_numpy(zs))
    _, g1 = gpu_pass(srcs, T, K48, W, H, nc, nf, eps, near, far, 1, zstar=zbuf, state=st)
    f = ro.samples(bt, o, d, src, ht, cnt, nc, 1, zs, eps, nf)
    assert f["totals"].sum() > 0
    assert np.array_equal(g1["totals"], f["totals"])
    assert np.array_equal(g1["points"].view(np.int32), f["points"].view(np.int32))
    assert np.array_equal(g1["z"].view(np.int32), f["z"].view(np.int32))
    used = f["counts"] > 0
    assert np.array_equal(g1["base"][used], f["base"][used])


def sphere_view(ens_list, bg=None):
    """Spheres trained at distinct world centres (CENTRES; the networks see world points, obj_center = 0), boxed
    around their centres and seen from z = -3; the background network is trained at the origin and boxed there."""
    centres = CENTRES
    srcs = []
    for i in range(4):
        e = ens_list[0]
        srcs.append(render.Source(e, i, i + 1, centres[i], np.eye(3), np.full(3, 0.7)))
    if bg is not None:
        srcs.append(render.Source(bg, 0, 0, np.zeros(3), np.eye(3), np.array([1.8, 1.4, 1.9])))
    T = np.eye(4)
    T[:3, 3] = [0.1, 0.0, -3.0]
    return srcs, T, centres


def rel(a, b, m=None):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if m is not None:
        a, b = a[m], b[m]
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


K40 = np.array([[48.0, 0, 19.5], [0, 48.0, 14.5], [0, 0, 1]])


def oracle_and_gpu(srcs, T, W, H, K, impl, nc=8, nf=4):
    out = ro.render(render.box_table(srcs), np.array([s.obj_id for s in srcs]), nets_of(srcs), W, H, K, T,
                    n_coarse=nc, n_fine=nf, eps=0.1, near=0.05, far=8.0)
    img, stats = render.render_view(srcs, T, K, W, H, n_coarse=nc, n_fine=nf, surface_eps=0.1, near=0.05, far=8.0,
                                    impl=impl)
    g = {k: v.cpu().numpy().reshape(W * H, -1).squeeze(-1) if k != "colour" else v.cpu().numpy().reshape(-1, 3)
         for k, v in img.items()}
    return out, g, stats


def test_full_view_fp32(ens32):
    srcs, T, _ = sphere_view([ens32])
    W, H = 40, 30
    out, g, stats = oracle_and_gpu(srcs, T, W, H, K40, "fp32")
    tie = np.abs(out["acc_at_surf"] - 0.5) < 1e-4
    ok = ~tie
    assert (out["instance"] >= 0).sum() > 100
    assert np.array_equal(g["coarse_surface"][ok], out["coarse_comp"]["surf"][ok])
    assert np.array_equal(g["instance"][ok], out["instance"][ok])
    for k in ("depth", "opacity", "colour"):
        assert rel(g[k], out[k], ok) < 1e-5, (k, rel(g[k], out[k], ok))
    assert stats["points_coarse"] == out["coarse"]["totals"].sum()


@pytest.mark.parametrize("bg_hidden", [None, 128, 256])
def test_full_view_tensor_cores(ens32, ens128, bg_hidden):
    bg = None if bg_hidden is None else (ens128 if bg_hidden == 128 else trained_ens(1, 256, steps=60, seed=3))
    srcs, T, _ = sphere_view([ens32], bg)
    W, H = 40, 30
    out, g, _ = oracle_and_gpu(srcs, T, W, H, K40, None)
    o0 = out["coarse_comp"]
    # rays whose coarse surface sample (index in the merged sequence) is the oracle's
    same = g["coarse_surface"] == o0["surf"]
    print(f"tensor cores (background hidden {bg_hidden}): same surface sample on {same.mean():.4f} of rays")
    assert (o0["surf"] >= 0).sum() > 100
    assert same.mean() >= 0.999, same.mean()
    for k in ("depth", "opacity", "colour"):
        assert rel(g[k], out[k], same) <= 1e-3, (k, rel(g[k], out[k], same))


def test_chunking_and_reproducible(ens32, ens128):
    srcs, T, _ = sphere_view([ens32], ens128)
    W, H = 96, 72                                          # 6912 rays: chunks of 4093 + 2819, of 1000 (6 + a tail)
    K = np.array([[90.0, 0, 47.5], [0, 90.0, 35.5], [0, 0, 1]])
    a, sa = render.render_view(srcs, T, K, W, H)
    b, sb = render.render_view(srcs, T, K, W, H)
    assert sa == sb and sa["points_fine"] > 0
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert int((a["instance"] >= 0).sum()) > 1000
    for chunk in (4093, 1000):
        c, sc = render.render_view(srcs, T, K, W, H, chunk_rays=chunk)
        assert sc == sa, chunk
        for k in a:
            assert torch.equal(a[k], c[k]), (chunk, k)


def test_empty_and_bad_arguments(ens32):
    T = np.eye(4)
    srcs = [render.Source(ens32, 0, 5, [0, 0, -4.0], np.eye(3), [0.5, 0.5, 0.5]),      # behind: empty segment
            render.Source(ens32, 1, 6, [40.0, 0, 2.0], np.eye(3), [0.5, 0.5, 0.5])]     # off-screen
    img, st = render.render_view(srcs, T, K48, 48, 36)
    assert st["points_coarse"] == 0 and st["points_fine"] == 0
    assert not img["depth"].any() and not img["opacity"].any() and not img["colour"].any()
    assert bool((img["instance"] == -1).all())
    good = dict(t_wc=T, K=K48, width=8, height=6)
    bad = [dict(width=0), dict(height=-1), dict(K=np.array([[0.0, 0, 1], [0, 1.0, 1], [0, 0, 1]])),
           dict(t_wc=np.full((4, 4), np.nan))]
    for b in bad:
        kw = {**good, **b}
        with pytest.raises(_lib.VmbError):
            render.render_view(srcs, kw["t_wc"], kw["K"], kw["width"], kw["height"])
    with pytest.raises(_lib.VmbError):
        render.render_view(srcs, T, K48, 8, 6, n_coarse=0)
    with pytest.raises(_lib.VmbError):
        render.render_view(srcs, T, K48, 8, 6, n_fine=-1)
    with pytest.raises(_lib.VmbError):
        render.render_view([render.Source(ens32, 0, 1, [0, 0, 2.0], np.eye(3), [0.5, 0.0, 0.5])], T, K48, 8, 6)
    with pytest.raises(_lib.VmbError):
        render.render_view([render.Source(ens32, 0, 1, [0, 0, np.inf], np.eye(3), [0.5, 0.5, 0.5])], T, K48, 8, 6)
    with pytest.raises(_lib.VmbError):
        render.render_view(srcs * 513, T, K48, 8, 6)


def analytic(centres, radii, T, K, W, H):
    o, d = ro.rays(W, H, K, T)
    best = np.full(W * H, np.inf)
    inst = np.full(W * H, -1)
    for i, (c, r) in enumerate(zip(centres, radii)):
        oc = o - c
        a = (d * d).sum(1)
        b = 2 * (d @ oc)
        cc = oc @ oc - r * r
        disc = b * b - 4 * a * cc
        t = np.where(disc >= 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
        closer = t < best
        best = np.where(closer, t, best)
        inst = np.where(closer, i + 1, inst)
    return inst.reshape(W, H), best.reshape(W, H)


def test_trained_spheres_quality():
    ens = trained_ens(4, 32, steps=300, seed=5, centres=CENTRES)
    srcs, T, centres = sphere_view([ens])
    W, H = 160, 120
    K = np.array([[120.0, 0, 79.5], [0, 120.0, 59.5], [0, 0, 1]])
    radii = 0.45 + 0.1 * np.arange(4) / 4
    inst, depth = analytic(centres, radii, T, K, W, H)
    core = np.ones_like(inst, bool)
    for du in range(-2, 3):
        for dv in range(-2, 3):
            core &= np.roll(np.roll(inst, du, 0), dv, 1) == inst
    core[:2], core[-2:], core[:, :2], core[:, -2:] = False, False, False, False
    fine, _ = render.render_view(srcs, T, K, W, H, n_coarse=32, n_fine=16, near=0.05, far=8.0)
    coarse, _ = render.render_view(srcs, T, K, W, H, n_coarse=32, n_fine=0, near=0.05, far=8.0)
    gi = fine["instance"].cpu().numpy()
    match = (gi == inst)[core].mean()
    on = core & (inst > 0)
    med_f = float(np.median(np.abs(fine["depth"].cpu().numpy() - depth)[on]))
    med_c = float(np.median(np.abs(coarse["depth"].cpu().numpy() - depth)[on]))
    print(f"trained spheres: instance match {match:.4f}, median |depth err| fine {med_f:.4f} coarse {med_c:.4f}")
    assert match >= 0.97
    assert med_f <= 0.02 and med_f <= med_c + 1e-6


def test_dropin_sources_from_objects(tmp_path):
    """Mirror API: sceneObjects with keyframes, the trained network, get_bound, then sources_from_objects and
    render_view from a keyframe pose; an object without bbox3d is left out and reported.  Then save_checkpoints and
    tools/eval_2d.py on a Replica-format directory reproduce the same images bitwise and write metrics_2D.npy."""
    from tests.test_mesh_gpu import R_SPHERE, _render_keyframes
    from vmap_b200 import cfg as cfg_mod
    from vmap_b200.vmap import sceneObject
    d = cfg_mod.replica_room0_dict()
    W, H = 96, 64
    d["camera"].update(w=W, h=H, fx=60.0, fy=60.0, cx=(W - 1) / 2, cy=(H - 1) / 2)
    d["model"]["keyframe_buffer_size"] = 8
    d["model"]["obj_scale"] = 2.0
    d["model"]["hidden_feature_size"] = 32
    d["trainer"]["do_bg"] = 0
    cfg = cfg_mod.Config(config_dict=d)
    frames, K = _render_keyframes(W, H, 60.0, 7, seed=3)
    objs = []
    for oid in (1, 2):
        obj = None
        for fid, (rgb, depth, inst, twc) in enumerate(frames):
            bbox = torch.tensor([0.0, W - 1.0, 0.0, H - 1.0], device="cuda")
            args = (rgb.cuda(), depth.cuda(), inst.to(torch.uint8).cuda(), bbox, twc.cuda())
            if obj is None:
                obj = sceneObject(cfg, oid, *args, fid)
            else:
                obj.append_keyframe(*args, frame_id=fid)
        objs.append(obj)
    ens = trained_ens(1, 32, steps=300, seed=7)          # sphere of radius 0.45 at the origin
    with torch.no_grad():
        for k, p in objs[0].trainer.fc_occ_map.named_parameters():
            p.copy_(ens.view(k)[0])
        objs[0].trainer.pe.B_layer.weight.copy_(ens.view("B_layer.weight")[0])
    from vmap_b200.lazy import ensemble_for_modules
    ensemble_for_modules(objs[0].trainer.fc_occ_map, objs[0].trainer.pe).refresh_image()
    assert objs[0].get_bound(K) is not None
    srcs, skipped = render.sources_from_objects(objs)
    assert skipped == [2] and len(srcs) == 1 and srcs[0].obj_id == 1
    assert np.allclose(srcs[0].half_extent, np.asarray(objs[0].bbox3d.extent) / (2 * 0.9))
    rgb, depth, inst, twc = frames[2]
    img, stats = render.render_view(srcs, twc, K, W, H, near=cfg.min_depth, far=cfg.max_depth,
                                    surface_eps=cfg.surface_eps)
    gi, gt_inst = img["instance"].cpu().numpy(), inst.numpy()
    agree = ((gi == 1) == (gt_inst == 1)).mean()
    on = (gt_inst == 1) & (gi == 1)
    err = float(np.median(np.abs(img["depth"].cpu().numpy() - depth.numpy())[on]))
    print(f"drop-in: silhouette agreement {agree:.4f}, median |depth err| {err:.4f} (sphere radius {R_SPHERE})")
    assert agree >= 0.95 and err <= 0.03
    # save_checkpoints -> tools/eval_2d.py on a cv2-written Replica directory
    import importlib.util
    import json
    import os
    import cv2
    root = tmp_path / "replica"
    (root / "rgb").mkdir(parents=True)
    (root / "depth").mkdir()
    for fid, (rgb_f, depth_f, _, _) in enumerate(frames):
        cv2.imwrite(str(root / "rgb" / f"rgb_{fid}.png"), cv2.cvtColor(rgb_f.numpy().transpose(1, 0, 2), cv2.COLOR_RGB2BGR))
        cv2.imwrite(str(root / "depth" / f"depth_{fid}.png"),
                    np.round(depth_f.numpy().T / cfg.depth_scale).astype(np.uint16))
    np.savetxt(str(root / "traj_w_c.txt"), np.stack([f[3].numpy().astype(np.float64).reshape(-1) for f in frames]))
    d["dataset"]["path"] = str(root)
    (tmp_path / "cfg.json").write_text(json.dumps(d))
    for obj in objs:
        os.makedirs(tmp_path / "ckpt" / str(obj.obj_id))
        obj.save_checkpoints(str(tmp_path / "ckpt" / str(obj.obj_id)), 5)
    spec = importlib.util.spec_from_file_location(
        "eval_2d", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "eval_2d.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    out = tmp_path / "eval"
    tool.main(["--config", str(tmp_path / "cfg.json"), "--ckpt-dir", str(tmp_path / "ckpt"), "--frame", "5",
               "--out", str(out), "--views", "2"])
    col = cv2.cvtColor(cv2.imread(str(out / "view_2_rgb.png")), cv2.COLOR_BGR2RGB).transpose(1, 0, 2)
    dmm = cv2.imread(str(out / "view_2_depth.png"), cv2.IMREAD_UNCHANGED).T
    ins = cv2.imread(str(out / "view_2_inst.png"), cv2.IMREAD_UNCHANGED).T
    assert np.array_equal(col, (img["colour"].clamp(0, 1) * 255).round().to(torch.uint8).cpu().numpy())
    assert np.array_equal(dmm.astype(np.int64), (img["depth"] * 1000).round().clamp(0, 65535).long().cpu().numpy())
    assert np.array_equal(ins.astype(np.int64), (img["instance"] + 1).long().cpu().numpy())
    m = np.load(str(out / "metrics_2D.npy"), allow_pickle=True)
    from vmap_b200.metrics import view_metrics
    gt_rgb = cv2.cvtColor(cv2.imread(str(root / "rgb" / "rgb_2.png")), cv2.COLOR_BGR2RGB).transpose(1, 0, 2)
    gt_d = cv2.imread(str(root / "depth" / "depth_2.png"), -1).astype(np.float32).T * np.float32(cfg.depth_scale)
    gt_d[gt_d > cfg.max_depth] = 0.0
    ref = view_metrics(img["colour"], img["depth"], torch.from_numpy(gt_rgb.astype(np.float32) / 255.0),
                       torch.from_numpy(gt_d))
    assert len(m) == 1 and m[0]["view"] == 2
    assert m[0]["psnr"] == ref["psnr"] and m[0]["depth_l1"] == ref["depth_l1"] and np.isfinite(ref["psnr"])
    # the tool re-renders from the checkpoints: bitwise the same images as the live objects
    srcs2, skipped2 = tool.load_sources(str(tmp_path / "ckpt"), 5)
    img2, _ = render.render_view(srcs2, twc, K, W, H, near=cfg.min_depth, far=cfg.max_depth, surface_eps=cfg.surface_eps)
    assert skipped2 == [2]
    for k in img:
        assert torch.equal(img[k], img2[k]), k
