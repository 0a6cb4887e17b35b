"""CPU restatement of vMAP's depth-guided ray sampler (vmap.py:319-459).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

The reference computes the per-ray sample depths by compacting rays into four
groups (invalid depth / valid / this-object / other-object) and drawing torch
randoms per group.  The CUDA sampler works per ray instead, so the restatement
is split the same way:

* ``draw_randoms_reference_order`` consumes a torch CPU generator in exactly
  the reference's call order and scatters the draws into *canonical per-ray
  arrays* (what the CUDA kernel takes in its injected-randoms mode);
* ``sample_from_randoms`` is the per-ray closed form evaluated from those
  arrays.

``tests/test_oracle_golden.py`` checks the pair against the reference's own
``sceneObject.get_training_samples`` run under the same seed.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch


@dataclass
class SamplerCfg:
    """The sceneObject fields the sampler reads (vmap.py:104-125)."""
    n_bins_cam2surface: int = 1     # room0_vMAP.json:28  (5 for bg / iMAP)
    n_bins: int = 9                 # room0_vMAP.json:27
    surface_eps: float = 0.1        # room0_vMAP.json:41
    stop_eps: float = 0.05          # room0_vMAP.json:42 ("other_eps")
    min_bound: float = 0.0          # render.depth_range[0]
    this_obj: int = 1               # vmap.py:148-150


def camera_ray_dirs(W: int, H: int, fx: float, fy: float, cx: float, cy: float) -> torch.Tensor:
    """cameraInfo.get_rays_dirs (vmap.py:507-524): [W,H,3] z-depth directions."""
    d = torch.ones(W, H, 3)
    d[:, :, 0] = ((torch.arange(W) - cx) / fx)[:, None]
    d[:, :, 1] = ((torch.arange(H) - cy) / fy)
    return d


def bin_limits(n: int) -> torch.Tensor:
    """torch.linspace(0,1,n+1) as stratified_bins builds it (vmap.py:48)."""
    return torch.linspace(0, 1, n + 1, dtype=torch.float32)


def draw_randoms_reference_order(gen: Optional[torch.Generator], n_keyframes: int,
                                 latest_kf: List[int], n_frames: int, n_samples: int,
                                 bbox: torch.Tensor, rgbs_batch: torch.Tensor,
                                 depth_batch: torch.Tensor, cfg: SamplerCfg) -> Dict[str, torch.Tensor]:
    """Consume randoms in the reference's order (vmap.py:321-346, 400-450) and
    return canonical per-ray arrays.  ``gen=None`` uses torch's global CPU
    generator (which is what the reference itself draws from)."""
    kw = {} if gen is None else {"generator": gen}
    n1, n2 = cfg.n_bins_cam2surface, cfg.n_bins
    if n_keyframes > 2:                                                     # :321-331
        kf = torch.randint(0, n_keyframes, (n_frames - 2,), dtype=torch.long, **kw)
        kf = torch.cat([kf, torch.tensor(latest_kf[-2:], dtype=torch.long)])
    else:                                                                   # :337-341
        kf = torch.randint(0, n_keyframes, (n_frames,), dtype=torch.long, **kw)
    u_w = torch.rand(n_frames, n_samples, **kw)                             # :343
    u_h = torch.rand(n_frames, n_samples, **kw)                             # :344
    iw, ih = pixel_indices(kf, u_w, u_h, bbox)
    state = rgbs_batch[kf[:, None], iw, ih][..., 3].reshape(-1)
    depth = depth_batch[kf[:, None], iw, ih].reshape(-1)
    n_rays = n_frames * n_samples
    invalid = depth <= cfg.min_bound                                        # :395
    valid = ~invalid
    this_m = (state == cfg.this_obj) & valid                                # :418
    other_m = (state != cfg.this_obj) & valid                               # :444
    u_z = torch.zeros(n_rays, n1 + n2)
    nrm = torch.zeros(n_rays, n2)
    if int(invalid.sum()):                                                  # :399-404
        u_z[invalid] = torch.rand(int(invalid.sum()), n1 + n2, **kw)
    if int(valid.sum()):                                                    # :411-415
        u_z[valid, :n1] = torch.rand(int(valid.sum()), n1, **kw)
        if int(this_m.sum()):                                               # :430-435, :81
            nrm[this_m] = torch.empty(int(this_m.sum()), n2).normal_(
                mean=0.0, std=cfg.surface_eps / 3.0, **kw)
        if int(other_m.sum()):                                              # :446-450
            u_z[other_m, n1:] = torch.rand(int(other_m.sum()), n2, **kw)
    return {"kf": kf, "u_w": u_w, "u_h": u_h, "u_z": u_z, "nrm": nrm}


def pixel_indices(kf: torch.Tensor, u_w: torch.Tensor, u_h: torch.Tensor, bbox: torch.Tensor, wh=None):
    """Uniforms -> integer pixel coordinates inside the keyframe's 2-D box
    (vmap.py:346-351): fp32 ``u*(hi-lo)+lo`` then truncation.  ``wh`` = (W, H):
    clamp to [0, W-1] x [0, H-1] as the CUDA sampler does for boxes that reach
    past the image.  The reference does not clamp: past the high border it indexes
    out of range, past the low border torch wraps the negative index to the
    opposite edge."""
    b = bbox[kf]                                   # [n_frames, 4] = u_lo,u_hi,v_lo,v_hi
    iw = (u_w * (b[:, 1] - b[:, 0])[:, None] + b[:, 0][:, None]).long()
    ih = (u_h * (b[:, 3] - b[:, 2])[:, None] + b[:, 2][:, None]).long()
    if wh is not None:
        iw, ih = iw.clamp(0, wh[0] - 1), ih.clamp(0, wh[1] - 1)
    return iw, ih


def _stratified(lo: torch.Tensor, hi: torch.Tensor, n: int, u: torch.Tensor) -> torch.Tensor:
    """stratified_bins (vmap.py:45-72) with the uniforms supplied: lo/hi [N], u [N,n]."""
    rng = hi - lo
    lower = rng[:, None] * bin_limits(n)[None, :-1] + lo[:, None]
    return lower + u * (rng / n)[:, None]


def sample_from_randoms(rnd: Dict[str, torch.Tensor], rgbs_batch: torch.Tensor,
                        depth_batch: torch.Tensor, t_wc_batch: torch.Tensor, bbox: torch.Tensor,
                        rays_dir: torch.Tensor, cfg: SamplerCfg):
    """Per-ray evaluation of get_training_samples + sample_3d_points
    (vmap.py:346-364, 366-459) from canonical randoms.

    Returns the reference's 6-tuple: rgb [F,P,3] u8, depth [F,P] f32,
    valid_depth_mask [F*P] bool, labels [F*P] u8, pcs [F,P,S,3] f32, z [F,P,S] f32."""
    kf, u_w, u_h = rnd["kf"], rnd["u_w"], rnd["u_h"]
    F_, P_ = u_w.shape
    n1, n2 = cfg.n_bins_cam2surface, cfg.n_bins
    eps, oeps = cfg.surface_eps, cfg.stop_eps
    iw, ih = pixel_indices(kf, u_w, u_h, bbox, wh=rgbs_batch.shape[1:3])
    px = rgbs_batch[kf[:, None], iw, ih]                     # [F,P,4] u8      :353
    depth = depth_batch[kf[:, None], iw, ih]                 # [F,P]           :354
    dirs_c = rays_dir[iw, ih]                                # [F,P,3]         :357
    twc = t_wc_batch[kf]                                     # [F,4,4]         :360
    origins = twc[:, :3, 3]                                  # vmap.py:39
    dirs_w = (twc[:, None, :3, :3] @ dirs_c[..., None]).squeeze(-1)   # vmap.py:37

    d = depth.reshape(-1)
    state = px[..., 3].reshape(-1)
    invalid = d <= cfg.min_bound
    valid = ~invalid
    this_m = (state == cfg.this_obj) & valid
    max_bound = d.max()                                      # :397 (data dependent)
    n_rays = d.numel()
    lo0 = torch.full((n_rays,), cfg.min_bound, dtype=torch.float32)

    z_inv = _stratified(lo0, torch.ones(n_rays) * max_bound, n1 + n2, rnd["u_z"])          # :401
    z_c2s = _stratified(lo0, d - eps, n1, rnd["u_z"][:, :n1])                              # :413
    bins = torch.clip(rnd["nrm"].sort(dim=-1).values, -eps, eps)                           # :81-82
    z_this = d[:, None] + bins                                                             # :83
    z_other = _stratified(d - eps, d + oeps, n2, rnd["u_z"][:, n1:])                       # :447
    z_val = torch.cat([z_c2s, torch.where(this_m[:, None], z_this, z_other)], dim=-1)
    z = torch.where(invalid[:, None], z_inv, z_val).view(F_, P_, n1 + n2)
    pcs = origins[:, None, None, :] + dirs_w[:, :, None, :] * z[..., None]                 # :455
    return px[..., :3], depth, valid, state.clone(), pcs, z
