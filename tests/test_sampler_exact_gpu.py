"""GPU: the ray sampler (K3) in Philox mode against the host restatement of its draws, output by output.

Reference: ``sampler_oracle.sample_from_randoms(philox_oracle.draw_randoms_philox(...))`` per object.  Pixels,
depths, colours, labels and masks are compared bitwise; z bitwise except on this-object rays, whose Box-Muller
normals go through the kernel's 1-ulp ``logf`` / ``sincospif`` (rows compared sorted, in ulps of z).  Points are
compared with origin + dir * z for the kernel's z, dir from fp64 and rounded once (the kernel forms it with an
``fmaf`` chain), in ulps of max(|origin|, sum_k |R_jk dc_k| * z): the magnitude the chain's terms carry, so that a
direction component that cancels to nearly zero does not turn a rounding of its terms into thousands of ulps.

Worst errors measured on an H100 over every case below: 1 ulp of z on this-object rays, 3.45 ulp on points.  Bars:
Z_ULP = 2 and PCS_ULP = 4 (4x the worst, capped at 4 ulp)."""
import numpy as np
import pytest
import torch

from oracle import philox_oracle as po
from oracle import sampler_oracle as so

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Z_ULP = 2.0
PCS_ULP = 4.0
EXACT_KEYS = ("gt_depth", "gt_colour", "gt_rgb_u8", "sem", "mask_depth")


# ---- fixtures --------------------------------------------------------------------------------------------------------
def _latest(n_kf):
    """Latest keyframes that are not (n_kf-2, n_kf-1), so taking them is observable."""
    return {1: [0, 0], 2: [1, 0], 3: [2, 0]}.get(n_kf, [n_kf - 2, 1])


def _boxes(KF, W, H, rng):
    """One box per keyframe, cycling through: fractional interior, the whole image, zero width, one pixel, and a box
    reaching past every border (the sampler clamps those pixels)."""
    out = []
    for k in range(KF):
        kind = k % 5
        if kind == 0:
            u0, v0 = rng.uniform(0, W / 2), rng.uniform(0, H / 2)
            out.append([u0, u0 + rng.uniform(1, W / 2), v0, v0 + rng.uniform(1, H / 2)])
        elif kind == 1:
            out.append([0, W, 0, H])
        elif kind == 2:
            out.append([W / 3 + 0.5, W / 3 + 0.5, 1.25, H - 1.5])
        elif kind == 3:
            out.append([7, 8, 3, 4])
        else:
            out.append([-3.5, W + 2.5, -1.25, H + 4.0])
    return torch.tensor(out, dtype=torch.float32)


def _poses(KF, rng):
    T = torch.zeros(KF, 4, 4)
    for k in range(KF):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        T[k, :3, :3] = torch.from_numpy(q * np.sign(np.linalg.det(q)))
        T[k, :3, 3] = torch.from_numpy(rng.uniform(-2, 2, 3))
    T[:, 3, 3] = 1
    return T


def make_objects(B, KF, W, H, n_kfs, min_bound, seed):
    """B objects (CPU tensors) with their own keyframes.  Object kinds cycle: mixed labels with zero / below-bound /
    exactly-at-bound depths, every pixel this object, no pixel this object, every depth invalid."""
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    rgbs = torch.randint(0, 256, (B, KF, W, H, 4), generator=g, dtype=torch.uint8)
    rgbs[..., 3] = torch.randint(0, 3, (B, KF, W, H), generator=g, dtype=torch.uint8)
    depth = torch.rand(B, KF, W, H, generator=g) * 3 + 0.5
    r = torch.rand(B, KF, W, H, generator=g)
    depth[r < 0.08] = 0
    depth[(r >= 0.08) & (r < 0.12)] = min_bound
    if min_bound > 0:
        depth[(r >= 0.12) & (r < 0.15)] = min_bound * 0.5
    objs = []
    for b in range(B):
        kind = b % 4 if B > 1 else 0
        if kind == 1:
            rgbs[b, ..., 3] = 1
        elif kind == 2:
            rgbs[b, ..., 3] = torch.where(rgbs[b, ..., 3] == 1, 2, rgbs[b, ..., 3])
        elif kind == 3:
            depth[b] = torch.rand(KF, W, H, generator=g) * min_bound
        nk = n_kfs[b % len(n_kfs)]
        objs.append((rgbs[b], depth[b], _poses(KF, rng), _boxes(KF, W, H, rng), nk, _latest(nk)))
    return objs


def kf_sets(objects):
    from vmap_b200.sampler import KeyframeSet
    return [KeyframeSet(r.to(DEV), d.to(DEV), t.to(DEV), bb.to(DEV), nk, lt) for r, d, t, bb, nk, lt in objects]


def rays_for(W, H):
    return so.camera_ray_dirs(W, H, 0.6 * W, 0.6 * W, W / 2 - 0.5, H / 2 - 0.5)


# ---- the comparator --------------------------------------------------------------------------------------------------
def _ulp(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def compare(got, objects, n_frames, n_pix, rays, cfg, seed, offset, b_index=None, **layout):
    """Assert the launch's outputs equal the restatement's; return the worst (z, pcs) ulp counts."""
    n1, n2 = cfg.n_bins_cam2surface, cfg.n_bins
    ref = po.sample_philox(objects, n_frames, n_pix, rays, cfg, seed, offset, b_index=b_index, **layout)
    got = {k: v.cpu() for k, v in got.items()}
    for k in EXACT_KEYS:
        if k in got:
            assert torch.equal(got[k], ref[k]), k
    this = (ref["mask_depth"] & (ref["sem"] == 1)).numpy()
    zg, zr = got["z"].numpy(), ref["z"].numpy()
    assert np.array_equal(zg[~this], zr[~this]), "z off this-object rays"
    assert np.array_equal(zg[this][:, :n1], zr[this][:, :n1]), "cam-to-surface z on this-object rays"
    a, b = np.sort(zg[this][:, n1:], axis=1), np.sort(zr[this][:, n1:], axis=1)
    z_ulp = float((np.abs(a.astype(np.float64) - b) / _ulp(b)).max()) if a.size else 0.0
    assert z_ulp <= Z_ULP, z_ulp
    # points: origin + dir * z with the kernel's z, fp64 directions rounded once to fp32
    pcs_ulp = 0.0
    for bi, (rgbs, depth, twc, bbox, n_kf, latest) in enumerate(objects):
        cb = bi if b_index is None else b_index[bi]
        rnd = po.draw_randoms_philox(seed, offset, cb, n_frames, n_pix, n_kf, latest, n1, n2, cfg.surface_eps, **layout)
        iw, ih = so.pixel_indices(rnd["kf"], rnd["u_w"], rnd["u_h"], bbox, wh=rgbs.shape[1:3])
        T = twc[rnd["kf"]].double()[:, None].expand(-1, n_pix, -1, -1).reshape(-1, 4, 4).numpy()
        dc = rays[iw, ih].double().reshape(-1, 3).numpy()
        dw = np.einsum("njk,nk->nj", T[:, :3, :3], dc).astype(np.float32).astype(np.float64)
        terms = np.einsum("njk,nk->nj", np.abs(T[:, :3, :3]), np.abs(dc))     # sum_k |R_jk dc_k| >= |dw_j|
        o = T[:, :3, 3]
        z = zg[bi].astype(np.float64)
        want = o[:, None, :] + dw[:, None, :] * z[:, :, None]
        unit = _ulp(np.maximum(np.abs(o)[:, None, :], terms[:, None, :] * np.abs(z)[:, :, None]))
        pcs_ulp = max(pcs_ulp, float((np.abs(got["pcs"][bi].numpy() - want) / unit).max()))
    assert pcs_ulp <= PCS_ULP, pcs_ulp
    return z_ulp, pcs_ulp


def chunks_per_object(B, N):
    """The sampler's grid: enough CTAs to fill the GPU a few times over (vmb_api.cu)."""
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    return max(min((N + 255) // 256, (8 * n_sm + B - 1) // B), 1)


# ---- Philox mode, per-object keyframes -------------------------------------------------------------------------------
# (n1, n2), B, n_frames, n_pix, n_kf per object (cycled), W, H, min_bound, seed, offset
CASES = {
    "t19_single_ray": ((1, 9), 1, 1, 1, [1], 64, 48, 0.0, 0, 0),
    "t59_one_cta": ((5, 9), 1, 3, 85, [3], 64, 48, 0.25, 2 ** 32 + 5, 1),
    "rt11_two_ctas": ((1, 1), 2, 2, 128, [7, 2], 64, 48, 0.0, 2 ** 63 - 1, 2 ** 31 + 7),
    "rt27_one_frame": ((2, 7), 3, 1, 257, [7, 3, 1], 64, 48, 0.25, 5, 0),
    "rt313_shipped_shape": ((3, 13), 20, 100, 24, [1, 2, 3, 7], 64, 48, 0.25, 2 ** 32 + 5, 2 ** 31 + 7),
    "rt131": ((1, 31), 3, 12, 40, [7, 3], 64, 48, 0.0, 2 ** 63 - 1, 1),
    "rt311": ((31, 1), 4, 3, 100, [3, 2, 7, 1], 64, 48, 0.25, 0, 2 ** 31 + 7),
    "s32_staging": ((16, 16), 3, 12, 64, [7, 1, 3], 64, 48, 0.0, 2 ** 32 + 5, 0),
    "t19_grid_stride_loop": ((1, 9), 200, 100, 48, [7, 3, 2, 1], 64, 48, 0.25, 5, 1),
    "rt1616_grid_stride_loop": ((16, 16), 200, 100, 24, [3, 7, 2, 1], 64, 48, 0.25, 2 ** 63 - 1, 1),
    "t19_max_obj": ((1, 9), 1024, 10, 100, [3, 7, 1, 2], 64, 48, 0.0, 2 ** 63 - 1, 2 ** 31 + 7),
    "t59_large_images": ((5, 9), 2, 3, 200, [3, 7], 1200, 680, 0.25, 0, 0),
    "t19_two_frames": ((1, 9), 4, 2, 70, [3, 7, 2, 1], 64, 48, 0.0, 7, 3),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_philox_draws_match_the_restatement(name):
    from vmap_b200.sampler import BatchedSampler
    (n1, n2), B, F, P, n_kfs, W, H, mb, seed, offset = CASES[name]
    objects = make_objects(B, max(n_kfs), W, H, n_kfs, mb, seed=sorted(CASES).index(name))
    rays = rays_for(W, H)
    smp = BatchedSampler(DEV, n_bins_cam2surface=n1, n_bins=n2, min_bound=mb)
    got = smp.sample(kf_sets(objects), F, P, rays.to(DEV), seed=seed, offset=offset, want_u8=True)
    cfg = so.SamplerCfg(n_bins_cam2surface=n1, n_bins=n2, min_bound=mb)
    z_ulp, pcs_ulp = compare(got, objects, F, P, rays, cfg, seed, offset)
    print(f"\n{name}: worst this-object z {z_ulp:.2f} ulp, pcs {pcs_ulp:.2f} ulp")
    if name.endswith("grid_stride_loop"):      # both passes loop: more 256-ray chunks than CTAs per object
        N = F * P
        assert (N + 255) // 256 > chunks_per_object(B, N), (N, chunks_per_object(B, N))
        print(f"{name}: {(N + 255) // 256} chunks over {chunks_per_object(B, N)} CTAs per object")


def test_offset_counter_on_the_device_equals_the_host_offset():
    from vmap_b200.sampler import BatchedSampler
    objects = make_objects(3, 7, 64, 48, [7, 3, 2], 0.0, seed=3)
    rays = rays_for(64, 48).to(DEV)
    smp = BatchedSampler(DEV)
    for k in (0, 5, 2 ** 31 + 7):
        a = {k_: v.clone() for k_, v in smp.sample(kf_sets(objects), 6, 30, rays, seed=9, offset=k).items()}
        b = smp.sample(kf_sets(objects), 6, 30, rays, seed=9, offset=123,
                       offset_dev=torch.tensor([k], dtype=torch.int64, device=DEV))
        for key in a:
            assert torch.equal(a[key], b[key]), (k, key)


def test_too_many_rays_per_object_is_an_argument_error():
    """Counter word 0 is ray * 8 + chunk: vmb_sample rejects n_frames * n_pix >= 2^29 (and products past int32).
    No output buffer is bound, so no launch can happen whatever the checks do: a launch of the legal size is refused
    for its missing outputs, and the oversized ones must be refused by the ray-count check."""
    import ctypes as C
    from vmap_b200 import _lib
    from vmap_b200.sampler import BatchedSampler, SamplerTables
    objects = make_objects(1, 1, 16, 12, [1], 0.0, seed=1)
    sets = kf_sets(objects)
    smp = BatchedSampler(DEV)
    tables = SamplerTables(DEV, 1)
    tables.fill_objects(sets)
    tables.upload()
    rays = rays_for(16, 12).to(DEV)
    for (F, P), why in (((4, 8), "missing tensor pointer"), ((2 ** 15, 2 ** 14), "2^29"), ((2 ** 16, 2 ** 16), "2^29")):
        a = _lib.SampleArgs()
        tables.bind(a)
        a.n_obj, a.n_frames, a.n_pix, a.n_bins_cam2surface, a.n_bins, a.width, a.height = 1, F, P, 1, 9, 16, 12
        a.rays_dir, a.bin_limits = C.c_void_p(rays.data_ptr()), C.c_void_p(smp.bin_limits.data_ptr())
        rc = smp.lib.vmb_sample(smp._handle, C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        msg = smp.lib.vmb_last_error(smp._handle).decode()
        assert rc == -1 and why in msg, (F, P, rc, msg)        # VMB_E_ARG
    torch.cuda.synchronize()


# ---- Philox mode, shared keyframe store ------------------------------------------------------------------------------
@pytest.mark.parametrize("n1,n2", [(5, 9), (2, 7)])
def test_store_mode_draws_match_the_restatement(n1, n2):
    """FrameStore + KeyframeTables, distinct object ids: the restatement runs on per-object copies whose state channel
    is derived from the instance image (this object -> 1, -1 -> 2, else 0)."""
    from vmap_b200.keyframes import FrameStore
    from vmap_b200.sampler import BatchedSampler, KeyframeTables
    W, H, n_store, KF, mb = 64, 48, 9, 7, 0.25
    rng = np.random.default_rng(n1 * 10 + n2)
    st = FrameStore(W, H, 12, DEV, max_id=64)
    frames = []
    for f in range(n_store):
        inst = torch.from_numpy(rng.integers(-1, 6, (W, H)).astype(np.int32))
        rgb = torch.from_numpy(rng.integers(0, 256, (W, H, 3), dtype=np.uint8))
        depth = torch.from_numpy((rng.random((W, H)) * 3 + 0.5).astype(np.float32))
        depth[torch.from_numpy(rng.random((W, H)) < 0.1)] = 0.0
        depth[torch.from_numpy(rng.random((W, H)) < 0.05)] = mb
        T = _poses(1, rng)[0]
        slot = st.put(rgb, depth, inst, T, frame_id=f)
        frames.append((slot, rgb, depth, inst, T))
    obj_ids, n_kf = [0, 3, 5, 1, 4], [7, 3, 2, 1, 5]
    B = len(obj_ids)
    kf_slot = np.zeros((B, KF), np.int32)
    kf_bbox = np.zeros((B, KF, 4), np.float32)
    objects = []
    for b, oid in enumerate(obj_ids):
        pick = rng.choice(n_store, KF, replace=False)
        bbox = _boxes(KF, W, H, rng)
        rgbs = torch.zeros(KF, W, H, 4, dtype=torch.uint8); deps = torch.zeros(KF, W, H); twc = torch.zeros(KF, 4, 4)
        for k, f in enumerate(pick):
            slot, rgb, depth, inst, T = frames[f]
            kf_slot[b, k], kf_bbox[b, k] = slot, bbox[k].numpy()
            rgbs[k, :, :, :3] = rgb
            rgbs[k, :, :, 3] = torch.where(inst == oid, 1, torch.where(inst == -1, 2, 0)).to(torch.uint8)
            deps[k], twc[k] = depth, T
        objects.append((rgbs, deps, twc, bbox, n_kf[b], _latest(n_kf[b])))
    tables = KeyframeTables(kf_slot, kf_bbox, obj_ids, n_kf, [_latest(n) for n in n_kf])
    smp = BatchedSampler(DEV, n_bins_cam2surface=n1, n_bins=n2, min_bound=mb)
    rays = rays_for(W, H)
    seed, offset = 2 ** 32 + 5, 2 ** 31 + 7
    got = smp.sample_store(st, tables, 10, 60, rays.to(DEV), seed=seed, offset=offset, want_u8=True)
    cfg = so.SamplerCfg(n_bins_cam2surface=n1, n_bins=n2, min_bound=mb)
    compare(got, objects, 10, 60, rays, cfg, seed, offset)
    assert set(torch.unique(got["sem"]).tolist()) == {0, 1, 2}


# ---- injected randoms on the run-time template -----------------------------------------------------------------------
@pytest.mark.parametrize("n1,n2", [(2, 7), (16, 16), (31, 1)])
def test_injected_randoms_on_the_run_time_template(n1, n2):
    from vmap_b200.sampler import BatchedSampler
    B, F, P, W, H, mb = 3, 5, 70, 64, 48, 0.25
    objects = make_objects(B, 7, W, H, [7, 3, 2], mb, seed=n1 + n2)
    g = torch.Generator().manual_seed(n1)
    S, N = n1 + n2, F * P
    inj = {"kf": torch.stack([torch.randint(0, o[4], (F,), generator=g) for o in objects]),
           "u_w": torch.rand(B, F, P, generator=g), "u_h": torch.rand(B, F, P, generator=g),
           "u_z": torch.rand(B, N, S, generator=g), "nrm": torch.randn(B, N, n2, generator=g) * 0.05}
    smp = BatchedSampler(DEV, n_bins_cam2surface=n1, n_bins=n2, min_bound=mb)
    rays = rays_for(W, H)
    got = smp.sample(kf_sets(objects), F, P, rays.to(DEV), inject=inj, want_u8=True)
    cfg = so.SamplerCfg(n_bins_cam2surface=n1, n_bins=n2, min_bound=mb)
    for b, (rgbs, depth, twc, bbox, _, _) in enumerate(objects):
        rnd = {k: v[b] for k, v in inj.items()}
        rgb, d, valid, lab, pcs, z = so.sample_from_randoms(rnd, rgbs, depth, twc, bbox, rays, cfg)
        assert torch.equal(got["z"][b].cpu(), z.reshape(N, S))
        assert torch.equal(got["sem"][b].cpu(), lab) and torch.equal(got["mask_depth"][b].cpu(), valid)
        assert torch.equal(got["gt_rgb_u8"][b].cpu(), rgb.reshape(N, 3))
        assert torch.equal(got["gt_depth"][b].cpu(), d.reshape(N))
        torch.testing.assert_close(got["pcs"][b].cpu(), pcs.reshape(N, S, 3), rtol=0, atol=5e-6)


# ---- the frame loop: device draw counter and the background key ------------------------------------------------------
def test_frame_loop_draws_match_the_restatement():
    """Frames 0-2 of a captured FrameLoop with a background model: objects draw at ``seed`` with offset
    first_offset + frame, the background at seed + 0x5bd1e995, (5, 9) bins, b = 0, from the same counter."""
    from vmap_b200 import synth
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.frame import Background, FrameLoop
    from vmap_b200.sampler import BatchedSampler
    B, KF, W, H, F, P, n_iter, seed, first = 3, 4, 64, 48, 8, 15, 4, 5, 7
    objects = make_objects(B, KF, W, H, [4, 3, 2], 0.0, seed=11)
    bg_obj = make_objects(1, KF, W, H, [4], 0.0, seed=12)
    rays = rays_for(W, H)
    ens = VmapEnsemble(B, hidden=32, scale=2.0, device=DEV)
    ens.load_stacked(synth.init_params(B, 32, seed=0))
    bg_ens = VmapEnsemble(1, hidden=128, scale=10.0, device=DEV)
    bg_ens.load_stacked(synth.init_params(1, 128, seed=1))
    bg = Background(bg_ens, BatchedSampler(DEV, 5, 9), n_frames=8, n_pix=10)
    fl = FrameLoop(ens, BatchedSampler(DEV, 1, 9), F, P, n_iter, rays.to(DEV), seed=seed, first_offset=first,
                   background=bg)
    sets, bg_sets = kf_sets(objects), kf_sets(bg_obj)       # the frame's tables hold their pointers: keep them alive
    fl.set_objects(sets)
    fl.set_background(bg_sets[0])
    for frame in range(3):
        fl.run()
        torch.cuda.synchronize()
        compare(fl.out, objects, F, P, rays, so.SamplerCfg(), seed, first + frame)
        compare(bg.out, bg_obj, 8, 10, rays, so.SamplerCfg(n_bins_cam2surface=5), seed + 0x5bd1e995, first + frame)
    assert int(fl.counter) == first + 3


# ---- the evaluation stream -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gt_key", [False, True])
def test_surface_sampler_stream_matches_the_restatement(gt_key):
    from vmap_b200.metrics import _GT_SEED_XOR, sample_surface
    from tests.test_eval_oracle import random_mesh
    v, f = random_mesh(5, nv=400, nf=2000)
    m = (v.astype(np.float32), f)
    seed = 2 ** 32 + 5
    if gt_key:
        seed ^= _GT_SEED_XOR
    N = 100000
    p, fi = sample_surface(m, N, seed=seed)
    q, fj = sample_surface(m, N, uniforms=po.surface_uniforms(seed, N))
    assert torch.equal(p, q) and torch.equal(fi, fj)
