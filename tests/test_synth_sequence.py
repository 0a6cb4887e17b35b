"""The synthetic sphere-room sequence: each depth pixel against the fp64 closed-form ray intersections, the instance and
class images against them, and the Replica writer read back with the reference loader's conventions."""
import os

import numpy as np
import pytest

from vmap_b200 import synth

W, H, F = 40, 30, 30.0


@pytest.fixture(scope="module")
def seq():
    return synth.sphere_room_sequence(12, W, H, F, F, W / 2 - 0.5, H / 2 - 0.5)


def _hits(T, spheres):
    """Per pixel, independently restated: every (z, instance) candidate of the spheres and room planes, nearest first."""
    out = np.empty((W, H), object)
    o = T[:3, 3]
    for u in range(W):
        for v in range(H):
            d = T[:3, :3] @ np.array([(u - (W / 2 - 0.5)) / F, (v - (H / 2 - 0.5)) / F, 1.0])
            c = []
            for (n0, n1, n2, h), i in zip(synth.ROOM_PLANES, synth.ROOM_IDS):
                n = np.array([n0, n1, n2], float)
                if n @ d != 0:
                    z = (h - n @ o) / (n @ d)
                    if z > 0:
                        c.append((z, i))
            for i, ctr, r in spheres:
                a, b, cc = d @ d, d @ (o - ctr), (o - ctr) @ (o - ctr) - r * r
                if b * b - a * cc >= 0:
                    z = (-b - np.sqrt(b * b - a * cc)) / a
                    if z > 0:
                        c.append((z, i))
            out[u, v] = sorted(c)
    return out


@pytest.mark.parametrize("k", [0, 6, 11])
def test_depth_instance_class_are_the_closed_form(seq, k):
    hits = _hits(seq["poses"][k], seq["spheres"])
    cls_of = dict(zip(synth.ROOM_IDS, synth.ROOM_CLASSES))
    for u in range(W):
        for v in range(H):
            z, i = hits[u, v][0]
            assert abs(seq["depth"][k, u, v] - z) <= 1e-12 * z
            assert seq["inst"][k, u, v] == i
            assert seq["cls"][k, u, v] == cls_of.get(i, synth.SPHERE_CLASS)
    p = seq["poses"][k][:3, 3] + seq["depth"][k][..., None] * (
        np.stack(np.meshgrid((np.arange(W) - (W / 2 - 0.5)) / F, (np.arange(H) - (H / 2 - 0.5)) / F, [1.0],
                             indexing="ij"), -1)[:, :, 0] @ seq["poses"][k][:3, :3].T)
    col = synth.sphere_room_colour(p, seq["inst"][k])
    assert np.array_equal(seq["rgb"][k], np.clip(np.round(col * 255), 0, 255).astype(np.uint8))


def test_sequence_shape_and_late_sphere(seq):
    assert seq["depth"].shape == (12, W, H) and seq["rgb"].shape == (12, W, H, 3)
    assert not (seq["inst"][0] == 4).any() and (seq["inst"][-1] == 4).any()
    assert all((seq["inst"][k] == i).any() for k in range(12) for i in (2, 3))
    assert np.allclose(seq["poses"][0], np.eye(4))
    R = seq["poses"][:, :3, :3]
    assert np.allclose(R @ R.transpose(0, 2, 1), np.eye(3), atol=1e-12)
    for k in range(12):                                  # colours vary across every surface
        assert seq["rgb"][k].reshape(-1, 3).std(0).min() > 5


def test_replica_writer_round_trip(seq, tmp_path):
    cv2 = pytest.importorskip("cv2")
    root = str(tmp_path)
    synth.write_replica(root, seq, depth_scale=1e-3)
    T = np.loadtxt(os.path.join(root, "traj_w_c.txt"), delimiter=" ").reshape([-1, 4, 4])     # dataset.py:67
    assert np.array_equal(T, seq["poses"])
    assert len(os.listdir(os.path.join(root, "depth"))) == 12
    for i in (0, 11):                                    # dataset.py:80-86
        depth = cv2.imread(os.path.join(root, "depth", f"depth_{i}.png"), -1).astype(np.float32).transpose(1, 0)
        image = cv2.cvtColor(cv2.imread(os.path.join(root, "rgb", f"rgb_{i}.png")).astype(np.uint8),
                             cv2.COLOR_BGR2RGB).transpose(1, 0, 2)
        obj = cv2.imread(os.path.join(root, "semantic_class", f"semantic_class_{i}.png"),
                         cv2.IMREAD_UNCHANGED).astype(np.int32).transpose(1, 0)
        inst = cv2.imread(os.path.join(root, "semantic_instance", f"semantic_instance_{i}.png"),
                          cv2.IMREAD_UNCHANGED).astype(np.int32).transpose(1, 0)
        assert np.max(np.abs(depth * np.float32(1e-3) - seq["depth"][i])) <= 0.5e-3 + 1e-6
        assert np.array_equal(image, seq["rgb"][i])
        assert np.array_equal(obj, seq["cls"][i]) and np.array_equal(inst, seq["inst"][i])
