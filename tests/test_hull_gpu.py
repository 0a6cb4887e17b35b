"""Exact convex hull and minimum-volume box on the GPU (K8): vertex sets against scipy's qhull, exact degeneracies,
facet structure, the device box against the host restatement of trimesh's oriented_bounds, and get_bound /
calc_3d_metric running with scipy's ConvexHull disabled."""
import tempfile
import types
from fractions import Fraction

import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull

from oracle import scannet_oracle as so

pytestmark = pytest.mark.gpu


def _hull(p):
    from vmap_b200.mesh import convex_hull
    h = convex_hull(torch.as_tensor(np.asarray(p, np.float64)).cuda())
    return h.vertices.cpu().numpy(), h.facets.cpu().numpy(), h.status


def _qhull_vertices(p):
    h = ConvexHull(p)
    assert len(h.coplanar) == 0                        # qhull merged nothing: its vertex set is the exact one
    return np.sort(h.vertices)


def _cloud(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "ball":
        x = rng.normal(size=(n, 3))
        return x / np.linalg.norm(x, axis=1, keepdims=True) * rng.uniform(0, 1, (n, 1)) ** (1 / 3)
    if kind == "cube":
        return rng.uniform(-1, 1, (n, 3))
    x = rng.normal(size=(n, 3))                         # noisy sphere shell
    return x / np.linalg.norm(x, axis=1, keepdims=True) * (1 + 1e-3 * rng.normal(size=(n, 1)))


# ---- exact checks ---------------------------------------------------------------------------------------------------
def _orient_sign(a, b, c, p):
    """sign det[b - a, c - a, p - a] for rows of a, b, c against every row of p: fp64 with a generous bound, exact
    rationals where the bound cannot decide.  Returns [len(a), len(p)]."""
    u, v = b - a, c - a
    n = np.cross(u, v)
    det = np.einsum("fk,fpk->fp", n, p[None, :, :] - a[:, None, :])
    scale = (np.abs(u).max(1) * np.abs(v).max(1))[:, None] * np.abs(p[None, :, :] - a[:, None, :]).max(2)
    s = np.sign(det).astype(np.int64)
    unsure = np.abs(det) <= 1e-12 * scale + 1e-300
    for f, q in zip(*np.nonzero(unsure)):
        A = [Fraction(x) for x in a[f]]
        U = [Fraction(x) - y for x, y in zip(b[f], A)]
        V = [Fraction(x) - y for x, y in zip(c[f], A)]
        W = [Fraction(x) - y for x, y in zip(p[q], A)]
        dd = (U[0] * (V[1] * W[2] - V[2] * W[1]) - U[1] * (V[0] * W[2] - V[2] * W[0])
              + U[2] * (V[0] * W[1] - V[1] * W[0]))
        s[f, q] = (dd > 0) - (dd < 0)
    return s


def _check_facets(p, vert, fac):
    """Every point on or below every facet (exact), every directed edge once and its reverse once, V - E + F = 2,
    and every extreme point is a facet corner."""
    assert len(fac) > 0
    s = _orient_sign(p[fac[:, 0]], p[fac[:, 1]], p[fac[:, 2]], p)
    assert (s <= 0).all()
    edges = np.concatenate([fac[:, [0, 1]], fac[:, [1, 2]], fac[:, [2, 0]]])
    fwd = {tuple(e) for e in edges.tolist()}
    assert len(fwd) == len(edges)
    assert all((b, a) in fwd for a, b in fwd)
    corners = np.unique(fac)
    assert len(corners) - len(edges) // 2 + len(fac) == 2
    assert set(vert.tolist()) <= set(corners.tolist())


# ---- 1. vertex sets equal qhull's -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,n", [("ball", 4), ("ball", 50), ("ball", 5000), ("ball", 200000), ("cube", 7),
                                    ("cube", 3000), ("cube", 200000), ("shell", 2000), ("shell", 60000)])
def test_vertices_match_qhull(kind, n):
    p = _cloud(kind, n, seed=n)
    ref = _qhull_vertices(p)
    vert, fac, st = _hull(p)
    assert st == 0
    np.testing.assert_array_equal(vert, ref)
    if n <= 5000:
        _check_facets(p, vert, fac)


def _oracle_clouds(seed, n_extra):
    """Every cloud the ScanNet oracle hands to the box fit on one synthetic sequence."""
    from oracle import o3d_standin
    seen = []
    orig = o3d_standin.obb_from_points

    def rec(points):
        seen.append(np.asarray(points, np.float64).reshape(-1, 3).copy())
        return orig(points)

    with tempfile.TemporaryDirectory() as root:
        so.write_sequence(root, seed=seed, n_frames=8, n_extra=n_extra, inf_frame=-1)
        o3d_standin.obb_from_points = rec
        try:
            so.run(root, n_trackers=1)
        finally:
            o3d_standin.obb_from_points = orig
    return seen


@pytest.mark.parametrize("seed,n_extra", [(3, 0), (5, 4), (7, 0), (11, 4)])
def test_scannet_oracle_clouds_contain_qhull_vertices(seed, n_extra):
    """Voxelised ScanNet clouds have nearly coplanar points that qhull's default facet merging drops from its vertex
    set without listing them as coplanar.  The exact vertex set holds every qhull vertex, and every extra one lies
    on qhull's hull within rounding."""
    from vmap_b200.mesh import convex_hull
    clouds = _oracle_clouds(seed, n_extra)
    assert len(clouds) > 10
    hulls = convex_hull([torch.from_numpy(c).cuda() for c in clouds])       # one launch for all of them
    for c, h in zip(clouds, hulls):
        if len(c) < 4:
            assert h.status == 1 and len(h.vertices) == 0
            continue
        assert h.status == 0
        got, q = h.vertices.cpu().numpy(), ConvexHull(c)
        assert set(q.vertices.tolist()) <= set(got.tolist())
        extra = np.setdiff1d(got, q.vertices)
        scale = np.abs(c).max()
        assert (np.abs(c[extra] @ q.equations[:, :3].T + q.equations[:, 3]).min(1) <= 1e-12 * scale).all()


def test_many_sets_in_one_launch():
    from vmap_b200.mesh import convex_hull
    rng = np.random.default_rng(1)
    sets = [np.zeros((0, 3)), rng.normal(size=(1, 3)), rng.normal(size=(3, 3)), _cloud("ball", 300, 2),
            np.zeros((0, 3)), _cloud("cube", 9000, 3), rng.normal(size=(4, 3)), _cloud("shell", 500, 4)]
    hulls = convex_hull([torch.from_numpy(s).cuda() for s in sets])
    for s, h in zip(sets, hulls):
        if len(s) < 4:
            assert h.status == 1 and len(h.vertices) == 0 and len(h.facets) == 0
        else:
            assert h.status == 0
            np.testing.assert_array_equal(h.vertices.cpu().numpy(), _qhull_vertices(s))
    # the sizes can come from a strided device table, as vmb_assoc_voxel's stats[:, 7]
    from vmap_b200.mesh import _hull_launch, _kernels
    pts = torch.from_numpy(np.concatenate(sets)).cuda()
    table = torch.zeros(len(sets), 8, dtype=torch.int32, device="cuda")
    table[:, 7] = torch.tensor([len(s) for s in sets], dtype=torch.int32)
    o = _hull_launch(_kernels(pts.device), pts, table[:, 7], 8, len(sets))
    vo = o["vertex_offset"].cpu().numpy()
    for i, h in enumerate(hulls):
        start = sum(len(s) for s in sets[:i])
        got = o["vertices"][vo[i]:vo[i + 1]].long().cpu().numpy() - start
        np.testing.assert_array_equal(got, h.vertices.cpu().numpy())


# ---- 2. exact degeneracies ------------------------------------------------------------------------------------------
def _lattice(k):
    g = np.arange(k, dtype=np.float64)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


def _corner_ids(p):
    lo, hi = p.min(0), p.max(0)
    return np.nonzero(((p == lo) | (p == hi)).all(1))[0]


def test_lattice_cube_has_only_its_corners():
    p = _lattice(6)                                     # 216 points: corners, edge, face and interior points
    vert, fac, st = _hull(p)
    assert st == 0
    np.testing.assert_array_equal(vert, _corner_ids(p))
    _check_facets(p, vert, fac)


def test_points_on_edges_and_faces_are_not_vertices():
    rng = np.random.default_rng(5)
    c = np.array([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)], np.float64)
    edge = np.array([[rng.integers(1, 8) / 8, 0, 0] for _ in range(10)])
    face = np.column_stack([rng.integers(1, 8, 10) / 8, rng.integers(1, 8, 10) / 8, np.ones(10)])
    p = np.concatenate([edge, face, c, face[:3] * [1, 1, 0]])
    vert, fac, st = _hull(p)
    assert st == 0
    np.testing.assert_array_equal(vert, np.arange(20, 28))
    _check_facets(p, vert, fac)


def test_duplicated_corners_flag_the_lowest_index():
    c = np.array([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)], np.float64)
    rng = np.random.default_rng(2)
    inner = rng.uniform(0.1, 0.9, (30, 3))
    p = np.concatenate([inner[:10], c[[5, 2]], inner[10:], c, c[[0, 7, 7]]])
    vert, _, st = _hull(p)
    assert st == 0
    first = {}
    for i, x in enumerate(map(tuple, p.tolist())):
        first.setdefault(x, i)
    np.testing.assert_array_equal(vert, sorted(first[tuple(x)] for x in c.tolist()))


@pytest.mark.parametrize("case", ["coplanar", "collinear", "identical", "tilted_plane"])
def test_flat_sets(case):
    rng = np.random.default_rng(3)
    if case == "coplanar":
        p = np.column_stack([rng.normal(size=(500, 2)), np.full(500, 0.25)])
    elif case == "collinear":
        p = np.outer(rng.integers(-50, 50, 300), [1.0, 2.0, -3.0])
    elif case == "identical":
        p = np.tile([[0.1, 0.2, 0.3]], (40, 1))
    else:                                                # exactly on x + 2y - z = 0 with integer coordinates
        xy = rng.integers(-1000, 1000, (9000, 2)).astype(np.float64)
        p = np.column_stack([xy, xy[:, 0] + 2 * xy[:, 1]])
    vert, fac, st = _hull(p)
    assert st == 2 and len(vert) == 0 and len(fac) == 0


@pytest.mark.parametrize("n", [0, 1, 2, 3])
def test_too_few(n):
    vert, fac, st = _hull(np.random.default_rng(n).normal(size=(n, 3)))
    assert st == 1 and len(vert) == 0 and len(fac) == 0


def test_tiny_set_far_from_origin_needs_the_exact_fallback():
    p = 1e3 + _lattice(5) * 2.0 ** -30                 # exact in fp64; face points have det exactly 0
    vert, fac, st = _hull(p)
    assert st == 0
    np.testing.assert_array_equal(vert, _corner_ids(p))
    _check_facets(p, vert, fac)


def test_integer_paraboloid_every_point_is_a_vertex():
    g = np.arange(-12, 13, dtype=np.float64)
    x, y = [a.ravel() for a in np.meshgrid(g, g, indexing="ij")]
    p = np.column_stack([x, y, x * x + y * y])
    p = p[np.random.default_rng(0).permutation(len(p))]
    vert, fac, st = _hull(p)
    assert st == 0
    np.testing.assert_array_equal(vert, np.arange(len(p)))
    _check_facets(p, vert, fac)


# ---- 4. device box vs host mesh.oriented_bounds ---------------------------------------------------------------------
def _host_volumes(pts):
    """Volume of the host fit's box for every distinct rounded normal (mesh.oriented_bounds' loop)."""
    from vmap_b200.mesh import _min_area_rect
    hull = ConvexHull(pts)
    hv = pts[hull.vertices]
    normals = hull.equations[:, :3] / np.linalg.norm(hull.equations[:, :3], axis=1, keepdims=True)
    vols = []
    for n in np.unique(np.round(normals, 10), axis=0):
        b1 = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0])
        b1 /= np.linalg.norm(b1)
        b2 = np.cross(n, b1)
        h = hv @ n
        vols.append(_min_area_rect(np.stack([hv @ b1, hv @ b2], 1))[0] * (h.max() - h.min()))
    return np.sort(vols)


def _box_cases():
    from tests.test_eval_oracle import uv_sphere
    rng = np.random.default_rng(9)
    A = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    return {"ball": _cloud("ball", 2000, 1), "cube": _cloud("cube", 3000, 2),
            "gauss": rng.normal(size=(3000, 3)) * [3.0, 1.0, 0.3] @ A.T, "shell": _cloud("shell", 1500, 3),
            "uv_sphere": uv_sphere(0.45, 30, 40)[0]}


@pytest.mark.parametrize("case", ["ball", "cube", "gauss", "shell", "uv_sphere"])
def test_box_matches_host_fit(case):
    from vmap_b200.mesh import oriented_bounds, oriented_bounds_gpu
    pts = _box_cases()[case]
    c0, R0, e0 = oriented_bounds(pts)
    c, R, e = oriented_bounds_gpu(torch.from_numpy(pts).cuda())
    assert abs(np.prod(e) / np.prod(e0) - 1) <= 1e-9
    assert np.allclose(R.T @ R, np.eye(3), atol=1e-9) and abs(np.linalg.det(R) - 1) < 1e-9   # n rounded to 1e-10
    loc = (pts - c) @ R
    assert (np.abs(loc) <= e / 2 + 1e-9).all()
    vols = _host_volumes(pts)
    if len(vols) > 1 and (vols[1] - vols[0]) > 1e-6 * vols[0]:
        P = np.abs(R0.T @ R)                            # same box up to axis order and sign
        assert np.allclose(np.sort(P, 0)[-1], 1, atol=1e-7)
        assert np.allclose(e, e0[P.argmax(0)], rtol=1e-9, atol=1e-12)
        assert np.allclose(c, c0, atol=1e-9)


@pytest.mark.parametrize("seed", range(5))
def test_box_recovers_rotated_box(seed):
    from tests.test_mesh_oracle import _rot
    from vmap_b200.mesh import oriented_bounds_gpu
    rng = np.random.default_rng(seed)
    ext = rng.uniform(0.2, 2.0, 3)
    R0, c0 = _rot(rng), rng.normal(size=3)
    corners = np.array([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)]) - 0.5
    local = np.concatenate([corners, rng.uniform(-0.5, 0.5, (500, 3))]) * ext
    pts = local @ R0.T + c0
    center, R, extent = oriented_bounds_gpu(pts)
    assert abs(np.linalg.det(R) - 1) < 1e-9
    assert np.allclose(R.T @ R, np.eye(3), atol=1e-9)
    assert np.allclose(center, c0, atol=1e-6)
    P = np.abs(R0.T @ R)
    assert np.allclose(np.sort(P, 1)[:, -1], 1, atol=1e-6)
    assert np.allclose(extent, ext[P.argmax(0)], atol=1e-6)
    assert (np.abs((pts - center) @ R) <= extent / 2 + 1e-9).all()


def test_box_degenerate_raises_value_error():
    from vmap_b200.mesh import oriented_bounds_gpu
    pts = np.random.default_rng(0).normal(size=(50, 3))
    pts[:, 2] = 0.0
    with pytest.raises(ValueError):
        oriented_bounds_gpu(pts)
    with pytest.raises(ValueError):
        oriented_bounds_gpu(pts[:3])


# ---- 5. no scipy hull on the three paths ----------------------------------------------------------------------------
@pytest.fixture
def no_qhull(monkeypatch):
    import scipy.spatial

    def refuse(*a, **k):
        raise AssertionError("scipy.spatial.ConvexHull called")

    return lambda: monkeypatch.setattr(scipy.spatial, "ConvexHull", refuse)


def test_get_bound_without_qhull(no_qhull):
    from tests.test_mesh_gpu import _render_keyframes
    from vmap_b200 import mesh
    from vmap_b200.vmap import sceneObject
    W, H = 96, 64
    frames, K = _render_keyframes(W, H, 60.0, 7, seed=3)
    state = torch.stack([f[2] for f in frames]).to(torch.uint8)
    o = types.SimpleNamespace(data_device="cuda:0", frames_width=W, frames_height=H, n_keyframes=7, obj_id=1,
                              store=None, kf_id_dict={}, bbox3d=None)
    o.rgbs_batch = torch.cat([torch.stack([f[0] for f in frames]), state[..., None]], -1).contiguous().cuda()
    o.depth_batch = torch.stack([f[1] for f in frames]).contiguous().cuda()
    o.t_wc_batch = torch.stack([f[3] for f in frames]).contiguous().cuda()
    pts = mesh.unproject_object(o, K).cpu().numpy().astype(np.float64)
    _, _, e0 = mesh.oriented_bounds(pts)
    no_qhull()
    bound = sceneObject.get_bound(o, K)
    assert bound is not None
    assert abs(np.prod(np.maximum(e0, 0.10)) / np.prod(bound.extent) - 1) <= 1e-9
    assert abs(np.linalg.det(bound.R) - 1) < 1e-9


def test_calc_3d_metric_crop_without_qhull(no_qhull):
    from tests.test_eval_oracle import uv_sphere
    from vmap_b200 import metrics
    from vmap_b200.mesh import oriented_bounds
    gv, gf = uv_sphere(0.45, 40, 80)
    rv, rf = uv_sphere(0.5, 30, 60)
    N = 20000
    rng = np.random.default_rng(0)
    u_rec, u_gt = rng.uniform(size=(N, 3)), rng.uniform(size=(N, 3))
    c, R, e = oriented_bounds(gv)
    soup = metrics.crop_to_box((rv, rf), c, R, e / 0.9)
    ref = metrics.calc_3d_metric(metrics.soup_mesh(soup), (gv, gf), N=N, uniforms=(u_rec, u_gt))
    no_qhull()
    got = metrics.calc_3d_metric((rv, rf), (gv, gf), N=N, crop_to_gt_box=True, uniforms=(u_rec, u_gt))
    assert got is not None
    for a, b in zip(got, ref):
        assert abs(a[0] - b[0]) <= 1e-9 * max(1.0, abs(b[0]))
