"""CPU tests of the ScanNet association restatement (oracle/scannet_oracle.py, oracle/o3d_standin.py): equal to the
reference's own dataset.ScanNet goldens, the erosion rule, stand-in properties and the new C struct layout."""
import os
import re
import tempfile

import cv2
import numpy as np
import pytest

from oracle import o3d_standin as o3d
from oracle import scannet_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_against_golden(g, results):
    assert len(results) == int(g["n_frames"])
    for i, (smp, tracks) in enumerate(results):
        np.testing.assert_array_equal(np.asarray(smp["obj"]), g[f"obj_{i}"], err_msg=f"frame {i} labels")
        keys = sorted(smp["bbox_dict"])
        assert keys == list(g[f"bbox_keys_{i}"]), i
        np.testing.assert_array_equal(np.stack([np.asarray(smp["bbox_dict"][k]).reshape(4) for k in keys]),
                                      g[f"bbox_{i}"])
        ids = sorted(tracks)
        assert ids == list(g[f"track_ids_{i}"]), i
        assert [tracks[k][3] for k in ids] == list(g[f"track_npts_{i}"]), i
        assert [tracks[k][4] for k in ids] == list(g[f"track_cmp_{i}"]), i
        for k, c, R, e in zip(ids, g[f"track_center_{i}"], g[f"track_R_{i}"], g[f"track_extent_{i}"]):
            np.testing.assert_allclose(tracks[k][0], c, rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(tracks[k][2], e, rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(np.abs(np.sum(tracks[k][1] * R, axis=0)), 1.0, atol=1e-9)


@pytest.mark.parametrize("name,n_trackers", [("seq", 1), ("workers", 4)])
def test_oracle_equals_reference_golden(golden_dir, name, n_trackers):
    g = np.load(os.path.join(golden_dir, f"ref_scannet_{name}.npz"))
    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=int(g["seed"]), n_frames=int(g["n_frames"]))
        check_against_golden(g, so.run(root, n_trackers=n_trackers))


def test_golden_sequence_covers_every_branch(golden_dir):
    g = np.load(os.path.join(golden_dir, "ref_scannet_seq.npz"))
    labels = [set(np.unique(g[f"obj_{i}"]).tolist()) for i in range(int(g["n_frames"]))]
    assert any(-1 in s for s in labels)                       # diff pixels / whole-mask -1
    assert labels[7] == {0}                                   # thin -1 strip relabelled 0
    assert 11 in labels[6] and 11 not in labels[8]            # A merged, then an 8-px sliver -> 0
    assert max(g["track_cmp_9"]) >= 8
    for missing in (13, 14, 15):                              # small, beyond max_depth, hull failure: never tracked
        assert missing not in g["track_ids_9"]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_cv2_erode_equals_clipped_13x13(seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 4, size=(6, 9)).repeat(9, 0).repeat(7, 1)      # blocky labels touching the border
    img = img[: 50 + seed, : 60 - seed]
    for lab in np.unique(img):
        m = img == lab
        ref = cv2.erode(m.astype(np.uint8), np.ones((5, 5)), iterations=3).astype(bool)
        np.testing.assert_array_equal(so.erode13(m), ref)


def test_obb_encloses_points_and_is_a_rotation():
    rng = np.random.default_rng(4)
    p = rng.normal(size=(500, 3)) * [0.5, 0.2, 0.1] @ o3d.np.linalg.qr(rng.normal(size=(3, 3)))[0] + [1, 2, 3]
    box = o3d.OrientedBoundingBox.create_from_points(p)
    np.testing.assert_allclose(box.R.T @ box.R, np.eye(3), atol=1e-12)
    assert abs(np.linalg.det(box.R) - 1.0) < 1e-12
    assert len(box.get_point_indices_within_bounding_box(p)) >= len(p) - 2       # hull points sit on the faces
    local = (p - box.center) @ box.R
    assert np.all(np.abs(local) <= box.extent / 2 + 1e-12)
    with pytest.raises(RuntimeError):
        o3d.OrientedBoundingBox.create_from_points(p[:3])


def test_voxel_means_equal_direct_mean():
    rng = np.random.default_rng(5)
    p = rng.uniform(-0.1, 0.1, size=(3000, 3))
    out = o3d.voxel_down_sample(p, 0.02)
    mb = p.min(0) - 0.01
    key = np.floor((p - mb) / 0.02).astype(np.int64)
    uk = np.unique(key, axis=0)                                  # ascending lexicographic, as the output
    assert len(out) == len(uk)
    for j, k in enumerate(uk):
        np.testing.assert_allclose(out[j], p[np.all(key == k, axis=1)].mean(0), rtol=0, atol=1e-15)


def test_unproject_matches_pinhole():
    d = np.zeros((4, 5), np.float32)
    d[1, 3], d[2, 0] = 2.0, 0.5
    P = np.eye(4)
    P[:3, 3] = [1, 2, 3]
    pts = o3d.unproject(d, 100.0, 200.0, 2.0, 1.5, P)
    np.testing.assert_allclose(pts, [[(3 - 2.0) * 2 / 100 + 1, (1 - 1.5) * 2 / 200 + 2, 5.0],
                                     [(0 - 2.0) * 0.5 / 100 + 1, (2 - 1.5) * 0.5 / 200 + 2, 3.5]])


def test_assoc_struct_matches_header_field_order():
    from vmap_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    body = src[src.index("typedef struct vmb_assoc_args"):src.index("} vmb_assoc_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"[\s\*]([a-z_0-9]+)\s*(?:\[\d+\])?\s*[;,]", body)
    assert names == [f[0] for f in _lib.AssocArgs._fields_]
    for n in ("vmb_assoc_classify", "vmb_assoc_voxel", "vmb_assoc_finalize"):
        assert n in _lib.EXPORTS
