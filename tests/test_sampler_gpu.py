"""GPU parity of the batched ray sampler (K3) through the C ABI."""
import os

import numpy as np
import pytest
import torch

from oracle import sampler_oracle as so
from tests._util import GOLDEN

pytestmark = pytest.mark.gpu


def _load(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    t = {k: torch.from_numpy(g[k]) for k in ("rgbs_batch", "depth_batch", "t_wc_batch", "bbox", "rays_dir")}
    return g, t


def _kfset(t, n_kf, latest, dev="cuda:0"):
    from vmap_b200.sampler import KeyframeSet
    return KeyframeSet(t["rgbs_batch"].to(dev), t["depth_batch"].to(dev), t["t_wc_batch"].to(dev),
                       t["bbox"].to(dev), n_kf, latest)


@pytest.mark.parametrize("name", ["sampler_obj", "sampler_bg", "sampler_2kf"])
def test_injected_randoms_reproduce_the_reference(name):
    """Same uniforms/normals as the reference drew -> identical pixels, labels, z; pcs to 1e-6."""
    from vmap_b200.sampler import BatchedSampler
    g, t = _load(name)
    n1, n_kf = int(g["n1"]), int(g["n_kf"])
    latest = [int(x) for x in g["latest"]]
    F, P = int(g["n_frames"]), int(g["n_samples"])
    cfg = so.SamplerCfg(n_bins_cam2surface=n1)
    torch.manual_seed(int(g["seed"]))
    rnd = so.draw_randoms_reference_order(None, n_kf, latest, F, P, t["bbox"], t["rgbs_batch"], t["depth_batch"], cfg)
    smp = BatchedSampler(n_bins_cam2surface=n1)
    # two identical objects in one launch: exercises the batched path
    objs = [_kfset(t, n_kf, latest), _kfset(t, n_kf, latest)]
    inj = {k: torch.stack([v, v]) for k, v in rnd.items()}
    out = smp.sample(objs, F, P, t["rays_dir"].cuda(), inject=inj, want_u8=True)
    for b in range(2):
        assert np.array_equal(out["gt_rgb_u8"][b].cpu().numpy().reshape(F, P, 3), g["o_rgb"])
        assert np.array_equal(out["gt_depth"][b].cpu().numpy().reshape(F, P), g["o_depth"])
        assert np.array_equal(out["mask_depth"][b].cpu().numpy(), g["o_valid"])
        assert np.array_equal(out["sem"][b].cpu().numpy(), g["o_lab"])
        assert np.array_equal(out["z"][b].cpu().numpy().reshape(g["o_z"].shape), g["o_z"])
        np.testing.assert_allclose(out["pcs"][b].cpu().numpy().reshape(g["o_pcs"].shape), g["o_pcs"], rtol=0, atol=1e-6)
        np.testing.assert_allclose(out["gt_colour"][b].cpu().numpy().reshape(F, P, 3), g["o_rgb"] / np.float32(255.))


def test_philox_mode_is_deterministic_and_distributionally_right():
    from vmap_b200.sampler import BatchedSampler
    g, t = _load("sampler_obj")
    n_kf, latest = int(g["n_kf"]), [int(x) for x in g["latest"]]
    F, P, n1, n2, eps, oeps = 100, 24, 1, 9, 0.1, 0.05
    smp = BatchedSampler(n_bins_cam2surface=n1)
    objs = [_kfset(t, n_kf, latest) for _ in range(3)]
    rd = t["rays_dir"].cuda()
    a = smp.sample(objs, F, P, rd, seed=123, offset=0)
    b = smp.sample(objs, F, P, rd, seed=123, offset=0)
    c = smp.sample(objs, F, P, rd, seed=123, offset=1)
    philox_mode_checks(a, b, c, n1, n2, eps, oeps)


def philox_mode_checks(a, b, c, n1, n2, eps, oeps):
    """The range / ordering / determinism checks of the Philox mode: ``a`` and ``b`` are two launches with the same
    seed and offset, ``c`` one at the next offset.  These alone do not pin which counter feeds which draw:
    tests/test_sampler_philox.py shows deliberately wrong draw schemes that pass them, and
    tests/test_sampler_exact_gpu.py compares the draws bit for bit."""
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert not torch.equal(a["z"], c["z"])
    assert not torch.equal(a["z"][0], a["z"][1])          # objects draw from different streams
    z = a["z"].cpu(); d = a["gt_depth"].cpu(); sem = a["sem"].cpu(); valid = a["mask_depth"].cpu()
    assert torch.equal(valid, d > 0)
    this_m = valid & (sem == 1)
    other_m = valid & (sem != 1)
    inv = ~valid
    maxb = d.max(dim=1, keepdim=True).values
    # cam-to-surface bin (vmap.py:413): [0, depth-eps)
    assert (z[..., 0][valid] >= 0).all() and (z[..., 0][valid] <= (d - eps)[valid] + 1e-6).all()
    # this-object: sorted, within +-eps of the surface (vmap.py:81-83)
    zt = z[..., n1:][this_m]
    assert (zt[:, 1:] >= zt[:, :-1]).all()
    assert ((zt - d[this_m][:, None]).abs() <= eps + 1e-6).all()
    assert 0.02 < float((zt - d[this_m][:, None]).std()) < 0.045        # sigma = eps/3
    # other-object: stratified over [depth-eps, depth+other_eps) (vmap.py:447)
    zo = z[..., n1:][other_m] - d[other_m][:, None]
    k = torch.arange(n2).float()
    assert (zo >= -eps + k * (eps + oeps) / n2 - 1e-5).all() and (zo <= -eps + (k + 1) * (eps + oeps) / n2 + 1e-5).all()
    # invalid depth: stratified over [0, max depth of the object's batch) (vmap.py:397-404)
    zi = z[inv]
    S = n1 + n2
    ks = torch.arange(S).float()
    mb = maxb.expand(-1, d.shape[1])[inv][:, None]
    assert (zi >= ks * mb / S - 1e-5).all() and (zi <= (ks + 1) * mb / S + 1e-5).all()
    # last two keyframe draws are the latest keyframes (vmap.py:321-331): their pixels come from those frames
    assert a["pcs"].isfinite().all()
    # uniform pixel choice inside the bbox: mean depth is plausible, labels cover all 3 states
    assert set(sem.unique().tolist()) == {0, 1, 2}
