"""CPU: the 3-D metric oracle (oracle/eval_oracle.py) against the reference's own metric/metrics.py
(tests/golden/ref_metrics.npz), the box crop and surface sampler on analytic cases, the mesh loaders of
vmap_b200.metrics, and the C structs of the K6 entry points."""
import os
import re
import struct

import numpy as np
import pytest

from oracle import eval_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- metrics vs the reference -------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", eo.METRIC_CASES, ids=[c[0] for c in eo.METRIC_CASES])
def test_oracle_metrics_equal_reference_golden(case, golden_dir):
    name, n_gt, n_rec, kind, seed = case
    g = np.load(os.path.join(golden_dir, "ref_metrics.npz"))
    gt, rec = eo.metric_points(n_gt, n_rec, kind, seed)
    assert np.array_equal(g[name + "_checksum"], [gt.sum(), rec.sum()])
    for key, val in (("accuracy", eo.accuracy(gt, rec)), ("completion", eo.completion(gt, rec)),
                     ("chamfer", eo.chamfer(gt, rec))):
        assert val == pytest.approx(float(g[name + "_" + key]), rel=1e-12, abs=0)
    assert eo.completion_ratio(gt, rec, 0.01) == float(g[name + "_ratio_0p01"])
    assert eo.completion_ratio(gt, rec, 0.05) == float(g[name + "_ratio_0p05"])


# ---- box crop -------------------------------------------------------------------------------------------------------
def uv_sphere(r=1.0, n_lat=120, n_lon=240):
    """Closed triangulated sphere: two poles and (n_lat - 1) rings of n_lon vertices."""
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.concatenate([[[0, 0, r]], np.stack([r * np.sin(T) * np.cos(P), r * np.sin(T) * np.sin(P), r * np.cos(T)],
                                              -1).reshape(-1, 3), [[0, 0, -r]]])
    ring = lambda i, j: 1 + i * n_lon + (j % n_lon)                          # noqa: E731
    f = [[0, ring(0, j), ring(0, j + 1)] for j in range(n_lon)]
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f += [[ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)], [ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)]]
    last = len(v) - 1
    f += [[ring(n_lat - 2, j), last, ring(n_lat - 2, j + 1)] for j in range(n_lon)]
    return v, np.asarray(f, np.int64)


def rot(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def random_mesh(seed, nv=300, nf=600):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(nv, 3)) * 0.5, rng.integers(0, nv, (nf, 3))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_clip_output_lies_in_box(seed):
    v, f = random_mesh(seed)
    R, c, ext = rot(seed + 10), np.array([0.1, -0.05, 0.02]), np.array([0.6, 0.9, 0.5])
    soup = eo.clip_to_box(v, f, c, R, ext)
    assert len(soup) > 50
    local = (soup.reshape(-1, 3) - c) @ R
    assert (np.abs(local) <= ext / 2 + 1e-9).all()


@pytest.mark.parametrize("rotated", [False, True])
def test_clip_sphere_zone_area(rotated):
    """A box that keeps the zone a < z' < b of a unit sphere (z' along one box axis) keeps the area 2 pi (b - a)."""
    v, f = uv_sphere()
    full = eo.soup_area(v[f])
    R = rot(3) if rotated else np.eye(3)
    a, b = -0.3, 0.55
    c = R @ np.array([0.0, 0.0, (a + b) / 2])
    soup = eo.clip_to_box(v, f, c, R, np.array([3.0, 3.0, b - a]))
    frac = eo.soup_area(soup) / full
    # the polyhedron's area deviates from the sphere's by O(h^2); the zone fraction to well under 1e-3
    assert frac == pytest.approx((b - a) / 2.0, abs=2e-3)
    local = (soup.reshape(-1, 3) - c) @ R
    assert local[:, 2].min() >= -(b - a) / 2 - 1e-9 and local[:, 2].max() <= (b - a) / 2 + 1e-9


def test_clip_inside_and_outside():
    v, f = random_mesh(4)
    R = rot(5)
    soup = eo.clip_to_box(v, f, np.zeros(3), R, np.full(3, 100.0))
    assert np.array_equal(soup, v[f])                                         # every face copied unchanged
    assert eo.soup_area(soup) == eo.soup_area(v[f])
    assert eo.clip_to_box(v, f, np.array([50.0, 0, 0]), R, np.full(3, 1.0)).shape == (0, 3, 3)


# ---- surface sampling -----------------------------------------------------------------------------------------------
def test_samples_lie_on_their_faces():
    v, f = random_mesh(6)
    pts, fi = eo.sample_surface(v, f, eo.uniforms(5000, 7))
    t = v[f[fi]]
    A = np.stack([t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]], -1)                  # [N, 3, 2]
    lam = np.stack([np.linalg.lstsq(A[i], pts[i] - t[i, 0], rcond=None)[0] for i in range(len(pts))])
    ok = eo.face_areas(v, f)[fi] > 1e-6
    assert (lam[ok] >= -1e-7).all() and (lam[ok].sum(1) <= 1 + 1e-7).all()
    assert np.abs((A @ lam[:, :, None])[:, :, 0] + t[:, 0] - pts).max() < 1e-9


def test_reflection_branch():
    v = np.array([[0.0, 0, 0], [1, 0, 0], [0, 2, 0]])
    f = np.array([[0, 1, 2]])
    u = np.array([[0.5, 0.25, 0.5], [0.5, 0.75, 0.5], [0.5, 0.9, 0.8]])
    pts, fi = eo.sample_surface(v, f, u)
    assert np.allclose(pts[0], [0.25, 1.0, 0])                               # u1 + u2 <= 1: as drawn
    assert np.allclose(pts[1], [0.25, 1.0, 0])                               # reflected: (1 - 0.75, 1 - 0.5)
    assert np.allclose(pts[2], [0.1, 0.4, 0])
    assert (fi == 0).all()


def test_face_counts_follow_area():
    from scipy.stats import chisquare
    rng = np.random.default_rng(8)
    v = rng.normal(size=(40, 3))
    f = rng.integers(0, 40, (25, 3))
    f = f[eo.face_areas(v, f) > 1e-3]
    a = eo.face_areas(v, f)
    N = 200000
    _, fi = eo.sample_surface(v, f, eo.uniforms(N, 9))
    obs = np.bincount(fi, minlength=len(f))
    assert chisquare(obs, N * a / a.sum()).pvalue > 1e-3
    # searchsorted(side='left'): u0 * total landing exactly on a boundary picks the face that ends there
    cum = np.cumsum(a)
    u = np.array([[cum[2] / cum[-1], 0.1, 0.1]])
    assert eo.sample_surface(v, f, u)[1][0] in (2, 3)


# ---- loaders --------------------------------------------------------------------------------------------------------
def test_export_load_roundtrip(tmp_path):
    from oracle import mesh_oracle as mo
    from vmap_b200.mesh import Mesh
    from vmap_b200.metrics import load_mesh
    x = np.linspace(-1, 1, 20)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    verts, faces, normals = mo.marching_cubes((0.6 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)).astype(np.float32), 0.0)
    m = Mesh(verts, faces, normals, np.full((len(verts), 4), 255, np.uint8))
    p = str(tmp_path / "frame_1999_obj3.obj")
    m.export(p)
    r = load_mesh(p)
    assert np.allclose(r.vertices, verts, atol=1e-6) and np.array_equal(r.faces, faces)


def _quad_mesh():
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0.5, 0.5, 1]], np.float64)
    polys = [[0, 1, 2, 3], [0, 1, 4], [1, 2, 4], [2, 3, 4], [3, 0, 4]]
    tris = [[0, 1, 2], [0, 2, 3], [0, 1, 4], [1, 2, 4], [2, 3, 4], [3, 0, 4]]
    return v, polys, np.array(tris)


def test_ascii_ply_quads_colours_and_face_attribute(tmp_path):
    from vmap_b200.metrics import load_mesh
    v, polys, tris = _quad_mesh()
    lines = ["ply", "format ascii 1.0", "comment hand-written", f"element vertex {len(v)}", "property float x",
             "property float y", "property float z", "property uchar red", "property uchar green", "property uchar blue",
             f"element face {len(polys)}", "property list uchar int vertex_indices", "property int object_id",
             "end_header"]
    lines += [f"{a} {b} {c} 10 20 30" for a, b, c in v]
    lines += [f"{len(p)} " + " ".join(map(str, p)) + f" {7 + i}" for i, p in enumerate(polys)]
    path = tmp_path / "m.ply"
    path.write_text("\n".join(lines) + "\n")
    m = load_mesh(str(path))
    assert np.allclose(m.vertices, v) and np.array_equal(m.faces, tris)


@pytest.mark.parametrize("uniform_lists", [False, True])
def test_binary_ply_quads_colours_and_face_attribute(tmp_path, uniform_lists):
    from vmap_b200.metrics import load_mesh
    v, polys, tris = _quad_mesh()
    if uniform_lists:                                             # all quads: the vectorised path
        polys, tris = [[0, 1, 2, 3], [3, 2, 1, 0]], np.array([[0, 1, 2], [0, 2, 3], [3, 2, 1], [3, 1, 0]])
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", "property double x",
            "property double y", "property double z", "property uchar red", "property uchar green",
            "property uchar blue", "property uchar alpha", f"element face {len(polys)}",
            "property list uchar int vertex_indices", "property int object_id", "end_header"]
    body = b"".join(struct.pack("<dddBBBB", *p, 1, 2, 3, 255) for p in v)
    body += b"".join(struct.pack("<B%diI" % len(p), len(p), *p, 40 + i) for i, p in enumerate(polys))
    path = tmp_path / "m.ply"
    path.write_bytes(("\n".join(head) + "\n").encode() + body)
    m = load_mesh(str(path))
    assert np.allclose(m.vertices, v) and np.array_equal(m.faces, tris)


def test_obj_polygon_and_index_forms(tmp_path):
    from vmap_b200.metrics import load_mesh
    path = tmp_path / "p.obj"
    path.write_text("v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nvt 0 0\nvn 0 0 1\nf 1/1/1 2/1/1 3/1/1 4/1/1\nf 1//1 3//1 -1//1\n")
    m = load_mesh(str(path))
    assert np.array_equal(m.faces, [[0, 1, 2], [0, 2, 3], [0, 2, 3]])


def test_concatenate_offsets_indices():
    from vmap_b200.metrics import TriangleMesh, concatenate
    a = TriangleMesh(np.zeros((3, 3)), [[0, 1, 2]])
    b = (np.ones((4, 3)), np.array([[0, 1, 2], [1, 2, 3]]))
    m = concatenate([a, b])
    assert m.vertices.shape == (7, 3) and np.array_equal(m.faces, [[0, 1, 2], [3, 4, 5], [4, 5, 6]])


# ---- C ABI ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c_name,py_name", [("vmb_clip_args", "ClipArgs"), ("vmb_surface_sample_args", "SurfaceSampleArgs"),
                                             ("vmb_nn_args", "NnArgs")])
def test_eval_structs_match_header_field_order(c_name, py_name):
    from vmap_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vmap_b200.h")).read()
    body = src[src.index("typedef struct " + c_name):src.index("} " + c_name + ";")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"[\s\*]([a-z_0-9]+)\s*(?:\[\d+\])?\s*[;,]", body)
    assert names == [f[0] for f in getattr(_lib, py_name)._fields_]
    for n in ("vmb_clip_count", "vmb_clip_emit", "vmb_surface_sample", "vmb_nn_dist"):
        assert n in _lib.EXPORTS
