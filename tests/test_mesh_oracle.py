"""CPU: the generated marching-cubes table, the oracle marching cubes on analytic and random volumes, the host box
fit of sceneObject.get_bound and Mesh.export."""
import numpy as np
import pytest

from oracle import mesh_oracle as mo


def test_committed_table_header_is_generator_output():
    with open(mo.HEADER) as f:
        assert f.read() == mo.header_text(), "regenerate with `python -m oracle.mesh_oracle`"


@pytest.mark.parametrize("case", range(256))
def test_case_cycles_follow_the_face_rule(case):
    ins = [(case >> c) & 1 for c in range(8)]
    cycles = mo.case_cycles(case)
    crossed = sorted(e for e, (c0, c1, _) in enumerate(mo.EDGES) if ins[c0] != ins[c1])
    assert sorted(e for cyc in cycles for e in cyc) == crossed          # every crossed edge on exactly one cycle
    for cyc in cycles:
        assert len(cyc) >= 3
    # segments of the cycles restricted to each face = the face rule (diagonal inside corners are separated)
    seg = {(cyc[i], cyc[(i + 1) % len(cyc)]) for cyc in cycles for i in range(len(cyc))}
    for a, s in mo.FACES:
        face_segs = set(mo._face_segments(case, a, s))
        assert face_segs <= seg
        corners = [c for c in range(8) if ((c >> a) & 1) == s]
        inside = [c for c in corners if ins[c]]
        n_cross = sum(1 for e, (c0, c1, ax) in enumerate(mo.EDGES)
                      if ax != a and ((c0 >> a) & 1) == s and ins[c0] != ins[c1])
        assert len(face_segs) == n_cross // 2
        if n_cross == 4:                                                 # each inside corner cut off on its own
            assert len(inside) == 2
            for c in inside:
                assert any(c in mo.EDGES[p][:2] and c in mo.EDGES[q][:2] for p, q in face_segs)
    ntri, tri = mo.make_table()
    t = tri[case, :ntri[case]]
    assert ntri[case] == sum(len(c) - 2 for c in cycles)
    assert all(len(set(row)) == 3 for row in t.tolist())               # no degenerate triangle in index space


def _grid(n, lo=-1.0, hi=1.0):
    x = np.linspace(lo, hi, n)
    return np.meshgrid(x, x, x, indexing="ij"), (hi - lo) / (n - 1)


def _check_closed(verts, faces):
    assert len(faces) > 0
    assert mo.directed_edge_check(faces)


@pytest.mark.parametrize("n", [32, 128])
def test_sphere(n):
    (X, Y, Z), h = _grid(n)
    r = 0.7
    v = (1.0 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2) / r).astype(np.float32)     # > 0 inside
    verts, faces, normals = mo.marching_cubes(v, 0.0)
    _check_closed(verts, faces)
    assert mo.euler_characteristic(verts, faces) == 2
    vol = mo.signed_volume(verts, faces) * h ** 3
    assert vol > 0
    if n == 128:
        assert abs(vol / (4 / 3 * np.pi * r ** 3) - 1) < 0.01
    # normals point outwards, i.e. along the position from the centre (in index units the centre is (n-1)/2)
    c = verts - (n - 1) / 2
    assert (np.einsum("ij,ij->i", c, normals) > 0).all()
    assert np.allclose(np.linalg.norm(normals, axis=1), 1, atol=1e-5)


@pytest.mark.parametrize("n", [48, 128])
def test_torus(n):
    (X, Y, Z), h = _grid(n)
    R, rr = 0.55, 0.25
    q = np.sqrt(X ** 2 + Y ** 2) - R
    v = (rr - np.sqrt(q ** 2 + Z ** 2)).astype(np.float32)
    verts, faces, _ = mo.marching_cubes(v, 0.0)
    _check_closed(verts, faces)
    assert mo.euler_characteristic(verts, faces) == 0
    vol = mo.signed_volume(verts, faces) * h ** 3
    assert vol > 0
    if n == 128:
        assert abs(vol / (2 * np.pi ** 2 * R * rr ** 2) - 1) < 0.01


def test_two_nearly_touching_spheres():
    (X, Y, Z), h = _grid(96)
    r, gap = 0.4, 1.5 * 2 / 95                 # 1.5 voxels apart: one grid plane between them is outside
    c = r + gap / 2
    d1 = np.sqrt((X - c) ** 2 + Y ** 2 + Z ** 2)
    d2 = np.sqrt((X + c) ** 2 + Y ** 2 + Z ** 2)
    v = np.maximum(r - d1, r - d2).astype(np.float32)
    verts, faces, _ = mo.marching_cubes(v, 0.0)
    _check_closed(verts, faces)
    assert mo.euler_characteristic(verts, faces) == 4      # two spheres
    assert mo.signed_volume(verts, faces) > 0


@pytest.mark.parametrize("seed", range(4))
def test_random_volume_every_case_closed(seed):
    rng = np.random.default_rng(seed)
    v = rng.random((17, 19, 23)).astype(np.float32)
    v[[0, -1]] = 0; v[:, [0, -1]] = 0; v[:, :, [0, -1]] = 0        # outside at the border: the surface closes
    ins = v > 0.5
    case = np.zeros((16, 18, 22), dtype=np.int64)
    for c in range(8):
        i, j, k = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= ins[i:16 + i, j:18 + j, k:22 + k].astype(np.int64) << c
    verts, faces, normals = mo.marching_cubes(v, 0.5)
    _check_closed(verts, faces)
    assert mo.signed_volume(verts, faces) > 0
    assert len(np.unique(case)) == 256
    # vertices lie on grid edges at the interpolated level crossing
    frac = verts - np.floor(verts)
    assert ((frac > 0).sum(1) <= 1).all()


def test_random_volumes_hit_every_case():
    seen = set()
    rng = np.random.default_rng(0)
    for _ in range(4):
        v = rng.random((17, 19, 23)) > 0.5
        case = np.zeros((16, 18, 22), dtype=np.int64)
        for c in range(8):
            i, j, k = c & 1, (c >> 1) & 1, (c >> 2) & 1
            case |= v[i:16 + i, j:18 + j, k:22 + k].astype(np.int64) << c
        seen |= set(np.unique(case).tolist())
    assert seen == set(range(256))


def test_affine_maps_vertices_and_normals():
    (X, Y, Z), _ = _grid(24)
    v = (0.6 - np.sqrt(X ** 2 + (Y * 1.3) ** 2 + Z ** 2)).astype(np.float32)
    rng = np.random.default_rng(3)
    Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if np.linalg.det(Q) < 0:
        Q[:, 0] = -Q[:, 0]
    A = np.concatenate([Q @ np.diag([0.5, 0.7, 0.9]), [[1.0], [-2.0], [0.5]]], 1)
    v0, f0, n0 = mo.marching_cubes(v, 0.0)
    v1, f1, n1 = mo.marching_cubes(v, 0.0, A)
    assert np.array_equal(f0, f1)
    assert np.allclose(v1, v0 @ A[:, :3].T + A[:, 3], atol=1e-5)
    assert mo.signed_volume(v1, f1) > 0


# ---- box fit -------------------------------------------------------------------------------------------------------
def _rot(rng):
    Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return Q if np.linalg.det(Q) > 0 else -Q


@pytest.mark.parametrize("seed", range(5))
def test_oriented_bounds_recovers_rotated_box(seed):
    from vmap_b200.mesh import oriented_bounds
    rng = np.random.default_rng(seed)
    ext = rng.uniform(0.2, 2.0, 3)
    R0, c0 = _rot(rng), rng.normal(size=3)
    corners = np.array([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)]) - 0.5
    local = np.concatenate([corners, rng.uniform(-0.5, 0.5, (500, 3))]) * ext
    pts = local @ R0.T + c0
    center, R, extent = oriented_bounds(pts)
    assert abs(np.linalg.det(R) - 1) < 1e-9
    assert np.allclose(R.T @ R, np.eye(3), atol=1e-9)
    assert np.allclose(center, c0, atol=1e-6)
    # same axes up to order and sign
    P = np.abs(R0.T @ R)
    assert np.allclose(np.sort(P, 1)[:, -1], 1, atol=1e-6)
    perm = P.argmax(0)
    assert np.allclose(extent, ext[perm], atol=1e-6)
    loc = (pts - center) @ R
    assert (np.abs(loc) <= extent / 2 + 1e-9).all()


def test_oriented_bounds_degenerate_raises():
    from scipy.spatial import QhullError
    from vmap_b200.mesh import oriented_bounds
    pts = np.random.default_rng(0).normal(size=(50, 3))
    pts[:, 2] = 0.0                                   # coplanar
    with pytest.raises(QhullError):
        oriented_bounds(pts)
    with pytest.raises(QhullError):
        oriented_bounds(pts[:3])


# ---- Mesh.export -----------------------------------------------------------------------------------------------------
def read_obj(path):
    v, c, n, f = [], [], [], []
    with open(path) as fh:
        for line in fh:
            t = line.split()
            if not t or t[0].startswith("#"):
                continue
            if t[0] == "v":
                v.append([float(x) for x in t[1:4]]); c.append([float(x) for x in t[4:7]])
            elif t[0] == "vn":
                n.append([float(x) for x in t[1:4]])
            elif t[0] == "f":
                f.append([int(x.split("/")[0]) - 1 for x in t[1:4]])
    return np.array(v), np.array(c), np.array(n), np.array(f)


def test_mesh_export_roundtrip(tmp_path):
    from vmap_b200.mesh import Mesh
    (X, Y, Z), _ = _grid(16)
    verts, faces, normals = mo.marching_cubes((0.6 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)).astype(np.float32), 0.0)
    rng = np.random.default_rng(0)
    rgba = np.concatenate([rng.integers(0, 256, (len(verts), 3)), np.full((len(verts), 1), 255)], 1).astype(np.uint8)
    m = Mesh(verts, faces, normals, rgba)
    p = str(tmp_path / "m.obj")
    m.export(p)
    v, c, n, f = read_obj(p)
    assert np.allclose(v, verts, atol=1e-6) and np.allclose(n, normals, atol=1e-6)
    assert np.array_equal(f, faces)
    assert np.array_equal(np.rint(c * 255).astype(np.uint8), rgba[:, :3])
    with pytest.raises(ValueError):
        m.export(str(tmp_path / "m.ply"))
