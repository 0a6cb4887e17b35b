"""Generate tests/golden/ref_*.npz: what tests/test_oracle_live_reference.py compares the oracle and the host mirror
against, produced by running the UNMODIFIED reference modules once (needs a reference checkout, see oracle/_refload.py;
no GPU; the loader case also needs cv2).

Run:  python -m oracle.make_reference_golden

Each ``ref_*`` function drives the reference exactly as the test drives the oracle (same seeds, same inputs) and
returns a dict of numpy arrays.  Large parameter tensors are stored as a fixed, seeded sample of their entries plus
their full L2 norm (``sample_index``).
"""
from __future__ import annotations

import json
import os
import random
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import _refload  # noqa: E402
from oracle import vmap_oracle as vo  # noqa: E402
from oracle import sampler_oracle as so  # noqa: E402
from oracle import ingest_oracle as io  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
N_SAMPLE = 256

STEP_CASES = [(1, 32, 17, 6, 2.0, 1, 21), (5, 32, 9, 10, 2.0, 1, 22), (2, 64, 13, 14, 5.0, 5, 23), (1, 128, 8, 10, 5.0, 5, 24),
              (3, 32, 1, 10, 2.0, 1, 25)]
SAMPLER_CASES = [(31, 7, 9, 11, 1), (32, 3, 6, 5, 5), (33, 1, 4, 7, 1), (34, 8, 20, 3, 1), (35, 4, 5, 16, 5)]
KEYFRAME_CASES = [(3, 6, 40, 1), (1, 4, 25, 2), (5, 8, 60, 3)]
LOADER_CASES = [(96, 64, 9, 41), (200, 150, 25, 42), (64, 96, 5, 43)]


def sample_index(numel: int, key: str) -> torch.Tensor:
    """The entries of a flattened tensor that the golden keeps (all of them when there are at most N_SAMPLE)."""
    if numel <= N_SAMPLE:
        return torch.arange(numel)
    g = torch.Generator().manual_seed(sum(key.encode()) + numel)
    return torch.randperm(numel, generator=g)[:N_SAMPLE]


def sampled(t: torch.Tensor, key: str) -> torch.Tensor:
    f = t.detach().reshape(-1)
    return f[sample_index(f.numel(), key)]


def _np(t):
    return t.detach().cpu().numpy().copy()


def step_inputs(n_obj, hidden, n_rays, n_samples, n_cam2surf, seed):
    """Initial parameters and batch of a step case: seeded, so the test regenerates them instead of storing them."""
    return (vo.init_params(n_obj, hidden, seed=seed),
            vo.synthetic_batch(n_obj, n_rays, n_samples, seed=seed + 100, n_cam2surf=n_cam2surf))


def ref_step(n_obj, hidden, n_rays, n_samples, scale, n_cam2surf, seed, n_steps=2):
    model, embedding, render_rays, loss = _refload.load("model", "embedding", "render_rays", "loss")
    from functorch import combine_state_for_ensemble, vmap
    init, batch = step_inputs(n_obj, hidden, n_rays, n_samples, n_cam2surf, seed)
    e1, e2 = vo.emb_sizes(5)
    fcs = [model.OccupancyMap(e1, e2, hidden_size=hidden) for _ in range(n_obj)]                            # trainer.py:27-33
    pes = [embedding.UniDirsEmbed(max_deg=5, scale=scale) for _ in range(n_obj)]
    for b in range(n_obj):
        fcs[b].load_state_dict({k: init[k][b].clone() for k in vo.FC_KEYS})
        with torch.no_grad():
            pes[b].B_layer.weight.copy_(init[vo.PE_KEY][b])
    opt = torch.optim.AdamW([torch.zeros(1, requires_grad=True)], lr=1e-3, weight_decay=0.013)             # train.py:67
    fc_model, fc_param, fc_buffer = combine_state_for_ensemble(fcs)                                        # utils.py:31
    pe_model, pe_param, pe_buffer = combine_state_for_ensemble(pes)
    for p in list(fc_param) + list(pe_param):
        p.requires_grad_()
    opt.add_param_group({"params": fc_param}); opt.add_param_group({"params": pe_param})
    names = [n for n, _ in fcs[0].named_parameters()]
    assert tuple(names) == vo.FC_KEYS

    def fwd_loss():
        emb = vmap(pe_model)(pe_param, pe_buffer, batch["pcs"])                                            # train.py:293
        alpha, col = vmap(fc_model)(fc_param, fc_buffer, emb)                                              # train.py:294
        return loss.step_batch_loss(alpha, col, batch["gt_depth"], batch["gt_colour"], batch["sem"],
                                    batch["mask_depth"], batch["z"])[0]                                    # train.py:303
    l0 = fwd_loss()
    l0.backward()
    grads = {n: p.grad.detach().clone() for n, p in zip(names, fc_param)}
    grads[vo.PE_KEY] = pe_param[0].grad.detach().clone()
    losses = [float(l0)]
    for s in range(n_steps):
        opt.step(); opt.zero_grad(set_to_none=True)
        l = fwd_loss(); losses.append(float(l))
        if s + 1 < n_steps:
            l.backward()
    final = {n: p.detach().clone() for n, p in zip(names, fc_param)}
    final[vo.PE_KEY] = pe_param[0].detach().clone()
    out = {"losses": np.asarray(losses, dtype=np.float64)}
    for k in vo.ALL_KEYS:
        out["init_" + k] = _np(sampled(init[k], k))          # guards the regenerated inputs
        out["g_" + k] = _np(sampled(grads[k], k)); out["gnorm_" + k] = np.float64(grads[k].double().norm())
        out["p_" + k] = _np(sampled(final[k], k)); out["pnorm_" + k] = np.float64(final[k].double().norm())
    return out


def sampler_inputs(seed, n_kf):
    W, H, KF = 56, 40, 8
    g = torch.Generator().manual_seed(seed)
    rgbs = torch.randint(0, 256, (KF, W, H, 4), generator=g).to(torch.uint8)
    rgbs[..., 3] = (torch.rand(KF, W, H, generator=g) * 3).long().clamp(0, 2).to(torch.uint8)
    depth = torch.rand(KF, W, H, generator=g) * 4 + 0.5
    depth[torch.rand(KF, W, H, generator=g) < 0.15] = 0.0
    twc = torch.eye(4).repeat(KF, 1, 1)
    twc[:, :3, 3] = torch.rand(KF, 3, generator=g) - 0.5
    bbox = torch.empty(KF, 4)
    bbox[:, 0] = torch.randint(0, W // 2, (KF,), generator=g).float()
    bbox[:, 1] = bbox[:, 0] + torch.randint(4, W // 2, (KF,), generator=g).float()
    bbox[:, 2] = torch.randint(0, H // 2, (KF,), generator=g).float()
    bbox[:, 3] = bbox[:, 2] + torch.randint(4, H // 2, (KF,), generator=g).float()
    rays = so.camera_ray_dirs(W, H, 60.0, 60.0, W / 2 - 0.5, H / 2 - 0.5)
    latest = [n_kf - 2, n_kf - 1] if n_kf >= 2 else [0]
    return rgbs, depth, twc, bbox, rays, latest


def ref_sampler(seed, n_kf, n_frames, n_samples, n1):
    vmap_mod = _refload.load("vmap")
    rgbs, depth, twc, bbox, rays, latest = sampler_inputs(seed, n_kf)
    obj = object.__new__(vmap_mod.sceneObject)          # skip __init__ (builds a Trainer / open3d)
    obj.n_keyframes, obj.data_device, obj.lastest_kf_queue = n_kf, "cpu", list(latest)
    obj.bbox, obj.rgbs_batch, obj.depth_batch, obj.t_wc_batch = bbox, rgbs, depth, twc
    obj.n_bins_cam2surface, obj.n_bins, obj.surface_eps, obj.stop_eps = n1, 9, 0.1, 0.05
    obj.min_bound, obj.max_bound = 0.0, 8.0
    obj.this_obj, obj.other_obj, obj.unknown_obj = 1, 0, 2
    obj.obj_center = torch.tensor(0.0)
    torch.manual_seed(seed + 1)
    names = ("rgb", "depth", "valid", "lab", "pcs", "z")
    return {n: _np(t) for n, t in zip(names, obj.get_training_samples(n_frames, n_samples, rays))}


def keyframe_cfg(kf_step, buf):
    return types.SimpleNamespace(do_bg=False, data_device="cpu", training_device="cpu", obj_scale=2.0, bg_scale=5.0,
                                 hidden_feature_size=32, hidden_feature_size_bg=128, n_bins_cam2surface=1,
                                 n_bins_cam2surface_bg=5, keyframe_step=kf_step, keyframe_step_bg=kf_step, min_depth=0.0,
                                 max_depth=8.0, n_bins=9, n_unidir_funcs=5, surface_eps=0.1, stop_eps=0.05,
                                 keyframe_buffer_size=buf)


KF_W, KF_H = 6, 5


def keyframe_frame(seed, fid):
    W, H = KF_W, KF_H
    g = torch.Generator().manual_seed(1000 * seed + fid)
    return (torch.randint(0, 255, (W, H, 3), dtype=torch.uint8, generator=g), torch.rand(W, H, generator=g),
            torch.randint(0, 3, (W, H), dtype=torch.uint8, generator=g), torch.tensor([0., float(fid % W), 0., float(fid % H)]),
            torch.eye(4) * (fid + 1))


def keyframe_state(o, buf):
    """One frame's observable state of a sceneObject (reference or mirror); buffer rows past the live ones are zeroed."""
    n = max(o.n_keyframes, (o.kf_pointer or 0) + 1)
    ids = np.full((2, buf + 1), -1, dtype=np.int64)
    for i, (k, v) in enumerate(sorted(dict(o.kf_id_dict).items())):
        ids[0, i], ids[1, i] = k, v
    q = np.full(4, -1, dtype=np.int64)
    q[:len(o.lastest_kf_queue)] = o.lastest_kf_queue
    scal = np.asarray([o.n_keyframes, -1 if o.kf_pointer is None else o.kf_pointer, o.frame_cnt, int(o.kf_buffer_full),
                       len(o.lastest_kf_queue), n], dtype=np.int64)

    def live(t):
        a = _np(t)
        a[n:] = 0
        return a
    return {"scal": scal, "ids": ids, "queue": q, "rgbs": live(o.rgbs_batch), "depth": live(o.depth_batch),
            "twc": live(o.t_wc_batch), "bbox": live(o.bbox)}


def ref_keyframes(kf_step, buf, n_frames_seen, seed):
    ref_mod = _refload.load("vmap")
    W, H = KF_W, KF_H
    rgb, depth, mask, bbox, T = keyframe_frame(seed, 0)
    ref = object.__new__(ref_mod.sceneObject)               # the reference __init__ builds a Trainer / needs open3d
    ref.n_keyframes, ref.kf_pointer, ref.keyframe_buffer_size = 1, None, buf
    ref.kf_id_dict, ref.kf_buffer_full, ref.frame_cnt, ref.lastest_kf_queue = _refload._Bidict({0: 0}), False, 0, []
    ref.keyframe_step, ref.rgb_idx, ref.state_idx = kf_step, slice(0, 3), slice(3, 4)
    ref.bbox = torch.zeros(buf, 4); ref.rgbs_batch = torch.zeros(buf, W, H, 4, dtype=torch.uint8)
    ref.depth_batch = torch.zeros(buf, W, H); ref.t_wc_batch = torch.zeros(buf, 4, 4)
    ref.bbox[0] = bbox; ref.rgbs_batch[0, :, :, :3] = rgb; ref.rgbs_batch[0, :, :, 3:4] = mask[..., None]
    ref.depth_batch[0] = depth; ref.t_wc_batch[0] = T
    frames = []
    for fid in range(1, n_frames_seen):
        rgb, depth, mask, bbox, T = keyframe_frame(seed, fid)
        random.seed(fid); ref.append_keyframe(rgb, depth, mask, bbox, T, fid)
        frames.append(keyframe_state(ref, buf))
    return {k: np.stack([f[k] for f in frames]) for k in frames[0]}


SURFACE_CAM = dict(data_device="cpu", W=37, H=23, fx=31.5, fy=29.25, cx=18.0, cy=11.5)


def ref_surface():
    ref_model, ref_emb, ref_vmap = _refload.load("model", "embedding", "vmap")
    sd = {str(h): [[k, list(v.shape)] for k, v in ref_model.OccupancyMap(87, 42, hidden_size=h).state_dict().items()]
          for h in (32, 128, 256)}
    pe = ref_emb.UniDirsEmbed(max_deg=5, scale=2.0)
    return {"occupancy_state_dict": np.asarray(json.dumps(sd)), "pe_keys": np.asarray(json.dumps(list(pe.state_dict()))),
            "pe_weight": _np(pe.B_layer.weight), "pe_scale": np.float64(float(pe.scale)),
            "rays_dir_cache": _np(ref_vmap.cameraInfo(types.SimpleNamespace(**SURFACE_CAM)).rays_dir_cache)}


def ref_loader(W, H, n_inst, seed):
    import cv2
    dataset = _refload.load("dataset")
    inst, cls = io.synthetic_instance_frame(W, H, n_inst, seed)
    root = tempfile.mkdtemp(prefix="_ds_")
    try:
        for d in ("rgb", "depth", "semantic_instance", "semantic_class"):
            os.makedirs(os.path.join(root, d))
        rng = np.random.default_rng(seed)
        cv2.imwrite(os.path.join(root, "rgb", "rgb_0.png"), rng.integers(0, 255, (H, W, 3), dtype=np.uint8))
        cv2.imwrite(os.path.join(root, "depth", "depth_0.png"), rng.integers(500, 4000, (H, W)).astype(np.uint16))
        cv2.imwrite(os.path.join(root, "semantic_instance", "semantic_instance_0.png"), inst.T.astype(np.uint16))
        cv2.imwrite(os.path.join(root, "semantic_class", "semantic_class_0.png"), cls.T.astype(np.uint16))
        np.savetxt(os.path.join(root, "traj_w_c.txt"), np.eye(4).reshape(1, 16), delimiter=" ")
        ds = dataset.Replica(types.SimpleNamespace(imap_mode=False, dataset_dir=root, depth_scale=1000.0, max_depth=8.0))
        sample = ds[0]
    finally:
        shutil.rmtree(root, ignore_errors=True)
    keys = sorted(int(k) for k in sample["bbox_dict"])
    boxes = np.asarray([[int(x) for x in np.asarray(sample["bbox_dict"][k]).reshape(-1)] for k in keys], dtype=np.int64)
    return {"bbox_keys": np.asarray(keys, dtype=np.int64), "bbox": boxes.reshape(len(keys), -1),
            "obj": np.asarray(sample["obj"]).astype(np.int32),
            "background_cls": np.asarray(sorted(ds.background_cls_list), dtype=np.int64), "bbox_scale": np.float64(ds.bbox_scale)}


def golden_path(kind, *case):
    return os.path.join(OUT, "ref_" + kind + "".join("_" + str(c).replace(".", "p") for c in case) + ".npz")


def main():
    for c in STEP_CASES:
        np.savez_compressed(golden_path("step", c[-1]), **ref_step(*c))
    for c in SAMPLER_CASES:
        np.savez_compressed(golden_path("sampler", c[0]), **ref_sampler(*c))
    for c in KEYFRAME_CASES:
        np.savez_compressed(golden_path("keyframes", c[-1]), **ref_keyframes(*c))
    np.savez_compressed(golden_path("surface"), **ref_surface())
    for c in LOADER_CASES:
        np.savez_compressed(golden_path("loader", c[-1]), **ref_loader(*c))
    for f in sorted(os.listdir(OUT)):
        if f.startswith("ref_"):
            print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
