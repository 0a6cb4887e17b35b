"""Oracle and host mirror vs the UNMODIFIED reference modules.  The reference side of every comparison was run once
by oracle/make_reference_golden.py (the same harness train.py uses: functorch vmap over combine_state_for_ensemble,
loss.step_batch_loss, torch.optim.AdamW; sceneObject.get_training_samples / append_keyframe; dataset.Replica) and is
replayed here from tests/golden/ref_*.npz, so the comparison runs wherever the repository does."""
import json
import random
import types

import numpy as np
import pytest
import torch

from oracle import make_reference_golden as mrg
from oracle import vmap_oracle as vo
from tests._util import rel_l2


def _golden(kind, *case):
    return np.load(mrg.golden_path(kind, *case))


@pytest.mark.parametrize("n_obj,hidden,n_rays,n_samples,scale,n1,seed", mrg.STEP_CASES)
def test_oracle_matches_live_reference_step(n_obj, hidden, n_rays, n_samples, scale, n1, seed):
    n_steps = 2
    G = _golden("step", seed)
    init, batch = mrg.step_inputs(n_obj, hidden, n_rays, n_samples, n1, seed)
    for k in vo.ALL_KEYS:                           # the regenerated inputs are the ones the reference ran on
        assert torch.equal(mrg.sampled(init[k], k), torch.from_numpy(G["init_" + k])), k
    l_ref = G["losses"]

    def check(mine, prefix, tol, k):
        ref_s, ref_n = torch.from_numpy(G[prefix + "_" + k]), float(G[prefix + "norm_" + k])
        assert rel_l2(mrg.sampled(mine, k), ref_s) < tol, k
        assert abs(float(mine.detach().double().norm()) - ref_n) <= tol * ref_n + 1e-12, k

    orc = vo.OracleEnsemble(init, scale)
    loss, grads = orc.grads(batch)
    assert abs(float(loss) - l_ref[0]) <= 2e-6 * abs(l_ref[0]) + 1e-7
    for k in vo.ALL_KEYS:
        check(grads[k], "g", 2e-5, k)
    orc = vo.OracleEnsemble(init, scale)            # fresh optimiser state / no leftover .grad
    losses = [float(orc.step(batch)) for _ in range(n_steps)]
    for a, b in zip(losses, l_ref[:n_steps]):
        assert abs(a - b) <= 5e-6 * abs(b) + 1e-7
    for k in vo.ALL_KEYS:
        check(orc.params[k], "p", 2e-6, k)


@pytest.mark.parametrize("seed,n_kf,n_frames,n_samples,n1", mrg.SAMPLER_CASES)
def test_sampler_oracle_matches_live_reference(seed, n_kf, n_frames, n_samples, n1):
    """sceneObject.get_training_samples (vmap.py:319-459) vs oracle/sampler_oracle.py with the reference's RNG
    call order reproduced: integer outputs and z bit-exact."""
    from oracle import sampler_oracle as so
    G = _golden("sampler", seed)
    rgbs, depth, twc, bbox, rays, latest = mrg.sampler_inputs(seed, n_kf)
    cfg = so.SamplerCfg(n_bins_cam2surface=n1)
    torch.manual_seed(seed + 1)
    rnd = so.draw_randoms_reference_order(None, n_kf, latest, n_frames, n_samples, bbox, rgbs, depth, cfg)
    rgb, dep, valid, lab, pcs, z = so.sample_from_randoms(rnd, rgbs, depth, twc, bbox, rays, cfg)
    for name, t in (("rgb", rgb), ("depth", dep), ("valid", valid), ("lab", lab), ("z", z)):
        ref = torch.from_numpy(G[name])
        assert t.dtype == ref.dtype and torch.equal(t, ref), name
    np.testing.assert_allclose(pcs.numpy(), G["pcs"], rtol=0, atol=1e-6)


@pytest.mark.parametrize("kf_step,buf,n_frames_seen,seed", mrg.KEYFRAME_CASES)
def test_keyframe_policy_matches_live_reference(kf_step, buf, n_frames_seen, seed, monkeypatch):
    """vmap_b200.vmap.sceneObject.append_keyframe / prune_keyframe vs the reference's (vmap.py:208-268), fed the same
    frames and the same ``random`` stream: slot choice, keyframe count, latest queue, id map and buffer contents."""
    from vmap_b200 import vmap as vm
    G = _golden("keyframes", seed)
    monkeypatch.setattr(vm.trainer_mod, "Trainer", lambda cfg: types.SimpleNamespace())
    rgb, depth, mask, bbox, T = mrg.keyframe_frame(seed, 0)
    mine = vm.sceneObject(mrg.keyframe_cfg(kf_step, buf), 7, rgb, depth, mask, bbox, T, 0)
    assert G["scal"].shape[0] == n_frames_seen - 1
    for fid in range(1, n_frames_seen):
        rgb, depth, mask, bbox, T = mrg.keyframe_frame(seed, fid)
        random.seed(fid); mine.append_keyframe(rgb, depth, mask, bbox, T, fid)
        st = mrg.keyframe_state(mine, buf)
        for k, v in st.items():
            assert np.array_equal(v, G[k][fid - 1]), (fid, k)


def test_module_surface_matches_live_reference():
    """state_dict keys / shapes of OccupancyMap and UniDirsEmbed, the icosahedron directions, and cameraInfo's ray cache
    against the reference classes (model.py:17-52, embedding.py:44-80, vmap.py:494-524)."""
    from vmap_b200 import embedding as my_emb, model as my_model, vmap as my_vmap
    G = _golden("surface")
    sd = json.loads(str(G["occupancy_state_dict"]))
    for hidden in (32, 128, 256):
        a = my_model.OccupancyMap(87, 42, hidden_size=hidden).state_dict()
        assert [[k, list(v.shape)] for k, v in a.items()] == sd[str(hidden)]
    pa = my_emb.UniDirsEmbed(max_deg=5, scale=2.0)
    assert list(pa.state_dict()) == json.loads(str(G["pe_keys"]))
    assert torch.equal(pa.B_layer.weight.detach(), torch.from_numpy(G["pe_weight"])) and float(pa.scale) == float(G["pe_scale"])
    cfg = types.SimpleNamespace(**mrg.SURFACE_CAM)
    assert torch.equal(my_vmap.cameraInfo(cfg).rays_dir_cache, torch.from_numpy(G["rays_dir_cache"]))


@pytest.mark.parametrize("W,H,n_inst,seed", mrg.LOADER_CASES)
def test_ingest_oracle_matches_live_reference_loader(W, H, n_inst, seed):
    """oracle/ingest_oracle.replica_frame vs dataset.Replica.__getitem__ (dataset.py:80-141) on a synthetic
    Replica-format frame."""
    from oracle import ingest_oracle as io
    G = _golden("loader", seed)
    inst, cls = io.synthetic_instance_frame(W, H, n_inst, seed)
    bbox_dict, obj = io.replica_frame(inst, cls, set(int(c) for c in G["background_cls"]), float(G["bbox_scale"]))
    ref_bbox = {int(k): [int(x) for x in row] for k, row in zip(G["bbox_keys"], G["bbox"])}
    assert {int(k): [int(x) for x in np.asarray(v).reshape(-1)] for k, v in bbox_dict.items()} == ref_bbox
    assert np.array_equal(obj, G["obj"])
