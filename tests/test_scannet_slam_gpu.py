"""Online SLAM on ScanNet-layout sequences (vmap_b200.slam with ``assoc``): the relabel kernel against the loader, the
mapping-only driver against the loader and a hand-driven loop, SLAM from GT frame 0 on the sphere room written in the
ScanNet layout (with a held-pose control), an invalid GT pose mid-sequence, reproducibility, graph replay, bundle
adjustment and tools/track_seq.py end to end."""
import importlib.util
import json
import os
import random
import tempfile

import numpy as np
import pytest
import torch

from oracle import scannet_oracle as so

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# 320 x 240: the spheres are 25-35 px in radius.  The reference's 1500 eroded pixels (13 x 13 erosion) would keep the
# smaller spheres out of the map at this size, so the tests pass min_pixels=400 to the association (and the loader).
W, H, FX, MW = 320, 240, 240.0, 10
N = 24
MIN_PIXELS = 400


def _cfg_dict(path, do_bg=False, imap=False):
    from vmap_b200.cfg import replica_room0_dict
    d = replica_room0_dict(imap=imap)
    d["dataset"].update(format="ScanNet", path=path)
    d["camera"] = {"w": W + 2 * MW, "h": H + 2 * MW, "mw": MW, "mh": MW}
    if not imap:
        d["trainer"]["do_bg"] = int(do_bg)
    return d


def _cfg(path, **kw):
    from vmap_b200.cfg import Config
    return Config(config_dict=_cfg_dict(path, **kw))


@pytest.fixture(scope="module")
def seq():
    from vmap_b200 import synth
    return synth.sphere_room_sequence(N, W, H, FX, FX, W / 2 - 0.5, H / 2 - 0.5)


@pytest.fixture(scope="module")
def data(seq, tmp_path_factory):
    from vmap_b200 import synth
    root = str(tmp_path_factory.mktemp("scannet_sphere_room"))
    synth.write_scannet(root, seq, mw=MW)
    return root


def _tracker(cfg):
    from vmap_b200.scannet import BBOX_SCALE, InstanceTracker
    return InstanceTracker(cfg.fx, cfg.fy, cfg.cx, cfg.cy, DEV, min_pixels=MIN_PIXELS, bbox_scale=BBOX_SCALE)


class _Record:
    """Per frame: the slot's relabelled instance image, the store's keep flags and boxes, and the keyframe tables."""

    def __init__(self, slam):
        self.slam, self.slots, self.labels, self.keep, self.bbox, self.tables = slam, [], [], [], [], []
        inner = slam.store.relabel

        def relabel(slot, labels, assoc_bbox):
            self.slots.append(slot)
            return inner(slot, labels, assoc_bbox)
        slam.store.relabel = relabel

    def after_step(self):
        from vmap_b200.vmap import keyframe_tables
        st = self.slam.store
        self.labels.append(st.inst[self.slots[-1]].cpu())
        self.keep.append(st.stats[:, 7].cpu())
        self.bbox.append(st.bbox.cpu())
        objs = list(self.slam.objects.values())
        self.tables.append(_tables(keyframe_tables(objs)) if objs else None)


def _tables(t):
    return [x.detach().cpu().clone() for x in (t.kf_slot, t.kf_bbox, t.obj_id, t.n_kf, t.latest)]


def _run(root, n=N, cfg=None, T_init=None, record=False, **kw):
    from vmap_b200 import scannet
    from vmap_b200.slam import Slam
    torch.manual_seed(0)
    random.seed(0)
    cfg = cfg or _cfg(root)
    frames = list(scannet.read_sequence(cfg, range(n)))
    T0 = frames[0]["T"] if T_init is None else T_init
    slam = Slam(cfg, T_init=T0, assoc=_tracker(cfg), max_frames=n, **kw)
    rec = _Record(slam) if record else None
    for f in frames:
        slam.step(f["rgb"], f["depth"], f["inst"], f["cls"], T_wc=f["T"])
        if rec is not None:
            rec.after_step()
    torch.cuda.synchronize()
    return slam, rec


# ---- the relabel kernel -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed,n_extra,id_base", [(3, 0, 10), (7, 20, 1030)])
def test_relabel_equals_the_loader(seed, n_extra, id_base):
    """FrameStore.relabel of the association's output gives the loader's obj / bbox_dict bit for bit, and clears every
    other row of the store's tables (which hold stale values from an earlier ingest here)."""
    from vmap_b200 import scannet
    from vmap_b200.cfg import Config
    from vmap_b200.keyframes import FrameStore
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=seed, n_frames=8, n_extra=n_extra, id_base=id_base)
        d = _cfg_dict(root)
        d["camera"] = {"w": 640, "h": 480, "mw": 10, "mh": 10}
        d["render"]["depth_range"] = [0.0, 6.0]
        cfg = Config(config_dict=d)
        loader = scannet.init_loader(cfg, shared_tracker=True)
        tracker = loader.dataset.trackers[0]
        store = FrameStore(cfg.W, cfg.H, 2, device=DEV)
        n_frames = 0
        for smp in loader:
            if smp is None:
                continue
            store.stats.fill_(7)
            store.bbox.fill_(3.5)
            slot = store.put(smp["image"], smp["depth"], torch.zeros(cfg.W, cfg.H, dtype=torch.int32), smp["T"].float())
            store.relabel(slot, smp["obj"], tracker.last_bbox)
            inst, stats, bbox = store.inst[slot].cpu(), store.stats.cpu(), store.bbox.cpu()
            store.release(slot)
            assert torch.equal(inst, smp["obj"].cpu().to(torch.int32))
            kept = sorted(k for k in smp["bbox_dict"] if k >= 0)
            assert torch.nonzero(stats[:, 7]).flatten().tolist() == kept
            assert torch.all(stats[:, :7] == 0)
            ref = torch.zeros_like(bbox)
            for k in kept:
                ref[k] = smp["bbox_dict"][k].to(torch.float32)
            assert torch.equal(bbox, ref)
            n_frames += 1
        assert n_frames >= 6
        assert any(k >= 1024 for k in tracker.inst_dict) == (id_base >= 1024)


# ---- the mapping-only driver --------------------------------------------------------------------------------------

def test_mapping_only_equals_the_loader_and_a_hand_loop(data, seq):
    """Slam(track=False, assoc=...) associates at the given pose, as the reference's train.py loop does with one
    tracker: the slot labels and boxes equal init_loader(shared_tracker=True)'s, and the keyframe tables and mapping
    losses equal the same parts driven by hand over those loader samples."""
    from vmap_b200 import scannet, utils
    from vmap_b200.frame import FrameLoop
    from vmap_b200.keyframes import FrameStore
    from vmap_b200.sampler import BatchedSampler
    from vmap_b200.track import _rays_dir
    from vmap_b200.vmap import keyframe_tables, sceneObject
    n = 12
    slam, rec = _run(data, n, track=False, graph=False, seed=3, record=True)
    res = slam.result()
    cfg = _cfg(data)
    loader = scannet.init_loader(cfg, shared_tracker=True)
    loader.dataset.trackers[0].min_pixels = MIN_PIXELS
    torch.manual_seed(0)
    random.seed(0)
    store = FrameStore(cfg.W, cfg.H, slam.store.capacity, device=DEV)
    smp_ = BatchedSampler(DEV, cfg.n_bins_cam2surface, cfg.n_bins, cfg.surface_eps, cfg.stop_eps, cfg.min_depth)
    rays = _rays_dir(cfg, torch.device(DEV))
    objs, loop, losses = {}, None, []
    opt = torch.optim.AdamW([torch.zeros((), requires_grad=True)], lr=cfg.learning_rate, weight_decay=cfg.weight_decay)
    for k, smp in enumerate(loader):
        if k == n:
            break
        obj = smp["obj"]
        assert torch.equal(rec.labels[k], obj.cpu().to(torch.int32)), k
        vis = {i: smp["bbox_dict"][i].to(torch.float32) for i in sorted(smp["bbox_dict"]) if i >= 0}
        assert torch.nonzero(rec.keep[k]).flatten().tolist() == sorted(vis), k
        for i, b in vis.items():
            assert torch.equal(rec.bbox[k][i], b), (k, i)
        T = smp["T"].float()
        slot = store.put(smp["image"], smp["depth"], obj, T, frame_id=k)
        new = False
        for i, bbox in vis.items():
            if i in objs:
                objs[i].append_keyframe(None, None, None, bbox, T, k, frame_slot=slot)
            else:
                objs[i] = sceneObject(cfg, i, None, None, None, bbox, T, k, store=store, frame_slot=slot)
                new = True
        if new:
            utils.update_vmap([o.trainer.fc_occ_map for o in objs.values()], opt)
            utils.update_vmap([o.trainer.pe for o in objs.values()], opt)
            old = loop
            loop = FrameLoop(opt._vmb_stack.ens, smp_, cfg.n_iter_per_frame * cfg.win_size, cfg.n_samples_per_frame,
                             cfg.n_iter_per_frame, rays, store=store, kf_stride=cfg.keyframe_buffer_size, seed=3)
            if old is not None:
                loop.counter.copy_(old.counter)
        tab = keyframe_tables(list(objs.values()))
        assert all(torch.equal(x, y) for x, y in zip(rec.tables[k], _tables(tab))), k
        loop.set_store_tables(tab)
        losses.append(float(loop.run_eager()[-1]))
        store.release(slot)
    torch.cuda.synchronize()
    assert list(objs) == list(slam.objects) and 1 in objs and 2 in objs
    assert np.array_equal(res["map_loss"], np.array(losses, np.float32)), (res["map_loss"], losses)
    assert torch.equal(slam.ens.params, opt._vmb_stack.ens.params)
    assert np.array_equal(res["poses"], seq["poses"][:n])


# ---- SLAM from GT frame 0 -----------------------------------------------------------------------------------------

# Bars (ATE rmse m, RPE m, RPE deg) per do_bg, from seeds 2 / 3 / 4 measured on an H100 80GB HBM3 (700 W), without and
# with bundle adjustment every 4 frames (ATE cm, RPE cm / deg):
#   do_bg on : 1.85 / 2.56 / 1.48 cm, RPE 0.69-0.80 cm / 0.23-0.30 deg; with BA 2.63 / 1.60 / 1.24 cm, RPE <= 1.23 cm /
#              0.37 deg.  Bars about twice the worst.  This test's run (seed 2, the store growing from 4 slots)
#              measured 3.69 cm, RPE 1.08 cm / 0.36 deg.
#   do_bg off: 7.72 / 9.41 / 5.89 cm, RPE 1.56-2.02 cm / 0.56-0.65 deg; with BA 3.93 / 7.86 / 5.23 cm, RPE <= 2.01 cm /
#              0.68 deg.  Tracking sees the spheres alone here and drifts; its bars sit between the worst run and the
#              held-pose control (ATE 12.5 cm, RPE 1.86 cm / 1.13 deg), which misses them.
BARS = {True: (0.05, 0.025, 0.75), False: (0.11, 0.025, 0.9)}


def _meets(ate, rpe, do_bg):
    a, t, r = BARS[do_bg]
    return ate["rmse"] < a and rpe["trans_rmse"] < t and rpe["rot_rmse_deg"] < r


def _slam_metrics(res, seq, n=N):
    from vmap_b200 import metrics
    valid = np.ones(n, bool)
    return (metrics.ate(res["poses"], seq["poses"][:n], valid=valid),
            metrics.rpe(res["poses"], seq["poses"][:n], valid=valid))


@pytest.mark.parametrize("do_bg", [False, True])
def test_slam_from_gt_frame_zero(data, seq, do_bg):
    slam, _ = _run(data, cfg=_cfg(data, do_bg=do_bg), track=True, graph=True, seed=2, store_capacity=4)
    res = slam.result()
    ate, rpe = _slam_metrics(res, seq)
    print(f"ScanNet SLAM do_bg={do_bg} {N} frames: ATE rmse {ate['rmse'] * 100:.3f} cm (max {ate['max'] * 100:.3f} "
          f"cm), RPE {rpe['trans_rmse'] * 100:.3f} cm / {rpe['rot_rmse_deg']:.3f} deg; inserted {res['inserted']}")
    assert np.array_equal(res["poses"][0], seq["poses"][0])
    assert not res["lost"].any()
    assert _meets(ate, rpe, do_bg)
    # the control: every frame held at T_0 misses the bars
    held = np.repeat(seq["poses"][:1], N, 0)
    ate0, rpe0 = _slam_metrics({"poses": held}, seq)
    assert ate0["rmse"] >= BARS[do_bg][0] and not _meets(ate0, rpe0, do_bg)
    # the late sphere is inserted partway and tracked from the next frame; the first three from frame 1
    assert 4 in res["inserted"] and 0 < res["inserted"][4] < N - 1
    assert 4 in res["tracked_ids"][res["inserted"][4] + 1]
    assert all(i in res["tracked_ids"][1] for i in (1, 2, 3))
    assert res["store_capacity"] > 4
    assert np.all(np.isfinite(res["track_loss"][1:])) and np.all(np.isfinite(res["map_loss"]))
    assert list(slam.phase_times()) == ["ingest", "track", "assoc", "bookkeeping", "map", "ba", "frame"]


def test_invalid_gt_pose_mid_sequence(seq, tmp_path):
    from vmap_b200 import metrics, synth
    n, bad = 14, 7
    root = str(tmp_path)
    synth.write_scannet(root, {k: (v[:n] if k in ("poses", "depth", "rgb", "inst", "cls") else v)
                               for k, v in seq.items()}, mw=MW, inf_frames=(bad,))
    from vmap_b200 import scannet
    from vmap_b200.slam import Slam
    torch.manual_seed(0)
    random.seed(0)
    cfg = _cfg(root)
    slam = Slam(cfg, T_init=seq["poses"][0], assoc=_tracker(cfg), max_frames=n, seed=2)
    gts = []
    for f in scannet.read_sequence(cfg):
        slam.step(f["rgb"], f["depth"], f["inst"], f["cls"])
        gts.append(f["T"])
    res = slam.result()
    gt = np.stack(gts)
    assert np.all(np.isinf(gt[bad])) and len(res["poses"]) == n
    assert not res["lost"].any() and np.all(np.isfinite(res["poses"][bad]))
    ate = metrics.ate(res["poses"], gt, valid=np.ones(n, bool))
    keep = [i for i in range(n) if i != bad]
    assert len(ate["errors"]) == n - 1
    assert ate["rmse"] == metrics.ate(res["poses"][keep], seq["poses"][keep])["rmse"]
    print(f"inf GT at frame {bad}: ATE rmse over the other frames {ate['rmse'] * 100:.3f} cm")
    assert ate["rmse"] < BARS[False][0]


def test_reproducible_graph_equals_eager_and_bundle_adjustment(data, seq):
    n = 10
    a, ra = _run(data, n, track=True, graph=True, seed=4, record=True)
    b, rb = _run(data, n, track=True, graph=True, seed=4, record=True)
    c, rc = _run(data, n, track=True, graph=False, seed=4, record=True)
    A, B, Cc = a.result(), b.result(), c.result()
    for X, rx in ((B, rb), (Cc, rc)):
        assert np.array_equal(A["poses"], X["poses"]), np.abs(A["poses"] - X["poses"]).max()
        assert np.array_equal(A["map_loss"], X["map_loss"])
        assert np.array_equal(A["track_loss"], X["track_loss"], equal_nan=True)
        assert all(torch.equal(p, q) for p, q in zip(ra.labels, rx.labels))
    assert "replay" in A["track_modes"] and "replay" not in Cc["track_modes"]
    slam, _ = _run(data, cfg=_cfg(data, do_bg=True), track=True, graph=True, seed=2, ba_every=4)
    res = slam.result()
    ate, rpe = _slam_metrics(res, seq)
    print(f"ScanNet SLAM with BA every 4: ATE rmse {ate['rmse'] * 100:.3f} cm, RPE {rpe['trans_rmse'] * 100:.3f} cm / "
          f"{rpe['rot_rmse_deg']:.3f} deg, passes {sum(1 for f in res['ba_frames'] if f)}")
    assert sum(1 for f in res["ba_frames"] if f) >= 4 and not res["lost"].any()
    assert _meets(ate, rpe, True)


# ---- tools/track_seq.py -------------------------------------------------------------------------------------------

def _tool():
    spec = importlib.util.spec_from_file_location("track_seq", os.path.join(ROOT, "tools", "track_seq.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("imap", [False, True])
def test_track_seq_tool_on_scannet(seq, tmp_path, capsys, imap):
    from vmap_b200 import metrics, synth
    n = 8
    root = str(tmp_path / "data")
    synth.write_scannet(root, {k: (v[:n] if k in ("poses", "depth", "rgb", "inst", "cls") else v)
                               for k, v in seq.items()}, mw=MW, inf_frames=(0, 5))
    cfg_file = str(tmp_path / "cfg.json")
    with open(cfg_file, "w") as f:
        json.dump(_cfg_dict(root, imap=imap), f)
    tool = _tool()
    out = tmp_path / "out"
    capsys.readouterr()
    tool.main(["--config", cfg_file, "--out", str(out), "--slam", "--frames", f"0:{n}"])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    print("imap" if imap else "vmap", line)
    est = np.loadtxt(out / "traj_est.txt", delimiter=" ").reshape(-1, 4, 4)
    assert est.shape == (n - 1, 4, 4)                       # the anchor is frame 1, the first with a GT pose
    assert np.array_equal(est[0], seq["poses"][1])
    m = np.load(out / "metrics_traj.npy", allow_pickle=True).item()
    assert m["frames"] == list(range(1, n)) and m["gt_invalid"] == [5] and line["gt_invalid"] == [5]
    keep = [i for i in range(1, n) if i != 5]
    ref = metrics.ate(est[[i - 1 for i in keep]], seq["poses"][keep])
    assert m["ate_aligned"]["rmse"] == ref["rmse"] and line["ate_rmse_m"] == ref["rmse"]
    assert ("assoc" in m["times_ms"]) == (not imap) and m["lost"] == []
    assert ref["rmse"] < 0.05
    with pytest.raises(SystemExit, match="ScanNet"):
        tool.main(["--config", cfg_file, "--out", str(out), "--ckpt-dir", str(tmp_path), "--frame", "1"])
