"""Handle scratch after a CUDA graph capture: the layer-wise tracking workspace (several buffers, and the activations of
a nested training-step workspace) keeps every buffer a captured tracker holds.  A larger call on the same handle is
refused with the capture error instead of moving a buffer under the graph; the graph still replays bit for bit, and
calls that fit still run."""
import math

import numpy as np
import pytest
import torch

from oracle import track_oracle as to
from oracle import vmap_oracle as vo

pytestmark = pytest.mark.gpu


def _rand_pose(seed, rot_deg=1.0, trans=0.02):
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3)
    w *= math.radians(rot_deg) / np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = to.exp_so3_np(w)
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _scene(hidden):
    """A 64 x 48 frame of three instances ingested into a FrameStore, and a small random hidden-64 / 128 map of them
    with its fp16 image (the layer-wise tracking path)."""
    from vmap_b200.cfg import Config, replica_room0_dict
    from vmap_b200.ensemble import VmapEnsemble
    from vmap_b200.keyframes import FrameStore
    d = replica_room0_dict()
    d["camera"].update(w=64, h=48, fx=40.0, fy=40.0, cx=31.5, cy=23.5)
    cfg = Config(config_dict=d)
    W, H = cfg.W, cfg.H
    g = torch.Generator().manual_seed(0)
    inst = torch.zeros(W, H, dtype=torch.int32)
    inst[5:25, 5:30] = 1
    inst[30:50, 10:40] = 2
    inst[40:60, 2:20] = 3
    depth = 1.0 + torch.rand(W, H, generator=g) * 2.0
    depth[::7, ::5] = 0.0
    rgb = torch.randint(0, 256, (W, H, 3), generator=g, dtype=torch.uint8)
    store = FrameStore(W, H, 4, device="cuda:0", max_id=16)
    slot, _, _ = store.ingest(rgb, depth, inst, torch.eye(4), min_extent=2)
    ens = VmapEnsemble(3, hidden=hidden, scale=2.0, impl="layerwise")
    ens.load_stacked(vo.init_params(3, hidden, seed=1))
    assert ens.image is not None
    return cfg, store, slot, [(ens, [1, 2, 3])]


@pytest.mark.parametrize("hidden", [64, 128])
def test_layerwise_tracking_scratch_after_a_capture(hidden):
    from vmap_b200 import _lib
    from vmap_b200.track import Tracker
    cfg, store, slot, groups = _scene(hidden)
    T0 = _rand_pose(4)
    ids = [1, 2, 3]
    kw = dict(n_iter=4, seed=3, impl="layerwise")
    eager = Tracker(groups, cfg, n_pix=40, **kw)
    graph = Tracker(groups, cfg, n_pix=40, **kw)
    assert graph.groups[0].lw
    p_eager, l_eager = eager.track(store, slot, T0, ids=ids)
    graph.capture(store, slot, T0, ids=ids)
    p_graph, l_graph = graph.run(store, slot, T0)
    torch.cuda.synchronize()
    assert torch.equal(p_graph, p_eager) and torch.equal(l_graph, l_eager)

    # more rays per iteration on the same ensemble (the same handle): every tracking buffer would have to grow
    with pytest.raises(_lib.VmbError, match="operation not permitted when stream is capturing"):
        Tracker(groups, cfg, n_pix=80, **kw).track(store, slot, T0, ids=ids)
    torch.cuda.synchronize()

    # the graph still holds its buffers: its second frame equals the eager tracker's second frame
    p_eager2, l_eager2 = eager.track(store, slot, T0, ids=ids)
    p_graph2, l_graph2 = graph.run(store, slot, T0)
    torch.cuda.synchronize()
    assert torch.equal(p_graph2, p_eager2) and torch.equal(l_graph2, l_eager2)
    assert not torch.equal(l_graph2, l_graph)                 # the draw counter moved on

    # a tracker at the captured size still runs on the handle, and reproduces the first frame
    p_again, l_again = Tracker(groups, cfg, n_pix=40, **kw).track(store, slot, T0, ids=ids)
    torch.cuda.synchronize()
    assert torch.equal(p_again, p_eager) and torch.equal(l_again, l_eager)
