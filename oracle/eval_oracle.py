"""CPU restatement of the 3-D reconstruction metrics (metric/metrics.py, eval_3D_obj.py, eval_3D_scene.py) in numpy /
scipy, the checker of the K6 kernels (csrc/k_eval.cuh) and vmap_b200/metrics.py.

- ``sample_surface``: trimesh.sample.sample_surface with the randoms injected (fp64 areas, cumsum, searchsorted
  side='left', reflected barycentrics).
- ``clip_to_box``: the crop of eval_3D_obj.py:12-15 as the kernel does it, per face Sutherland-Hodgman against the
  box's six half-spaces and a fan from the first vertex, in fp64, so the GPU soup can be compared triangle for triangle.
- ``accuracy`` / ``completion`` / ``completion_ratio`` / ``chamfer``: metric/metrics.py via scipy's cKDTree.
- ``calc_3d_metric``: eval_3D_*.calc_3d_metric with injected uniforms.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree


# ---- metric/metrics.py ----------------------------------------------------------------------------------------------
def _nn(ref, query):
    return cKDTree(np.asarray(ref, np.float64)).query(np.asarray(query, np.float64))[0]


def accuracy(gt_points, rec_points):
    return float(np.mean(_nn(gt_points, rec_points)))


def completion(gt_points, rec_points):
    return float(np.mean(_nn(rec_points, gt_points)))


def completion_ratio(gt_points, rec_points, dist_th=0.01):
    return float(np.mean((_nn(rec_points, gt_points) < dist_th).astype(np.float64)))


def chamfer(gt_points, rec_points):
    return (completion(gt_points, rec_points) + accuracy(gt_points, rec_points)) / 2.0


# Seeded point sets the reference's metrics are run on (tests/golden/ref_metrics.npz): (name, n_gt, n_rec, kind, seed)
METRIC_CASES = [("uniform", 1500, 1200, "uniform", 1), ("blobs", 800, 2000, "blobs", 2),
                ("sphere", 3000, 2500, "sphere", 3), ("tiny", 1, 7, "uniform", 4)]


def metric_points(n_gt, n_rec, kind, seed):
    """(gt [n_gt,3], rec [n_rec,3]) float64; rec is gt's distribution perturbed so the ratios are neither 0 nor 1."""
    rng = np.random.default_rng(seed)
    centers = rng.normal(size=(4, 3)) * 0.5

    def draw(n):
        if kind == "uniform":
            return rng.random((n, 3)) * 0.3
        if kind == "blobs":                                      # four tight blobs and 2 % far outliers
            p = centers[rng.integers(0, 4, n)] + rng.normal(size=(n, 3)) * 0.02
            far = rng.random(n) < 0.02
            p[far] = rng.normal(size=(int(far.sum()), 3)) * 5.0
            return p
        d = rng.normal(size=(n, 3))
        return 0.4 * d / np.linalg.norm(d, axis=1, keepdims=True)
    gt = draw(n_gt)
    rec = draw(n_rec) + rng.normal(size=(n_rec, 3)) * 0.01
    return gt, rec


# ---- trimesh.sample.sample_surface --------------------------------------------------------------------------------
def face_areas(vertices, faces):
    t = np.asarray(vertices, np.float64)[np.asarray(faces, np.int64)]
    c = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    return np.sqrt((c ** 2).sum(axis=1)) / 2.0


def sample_surface(vertices, faces, uniforms):
    """(points [N,3] f64, face_index [N] int64) for uniforms [N,3] = (u0, u1, u2)."""
    u = np.asarray(uniforms, np.float64)
    cum = np.cumsum(face_areas(vertices, faces))
    fi = np.minimum(np.searchsorted(cum, u[:, 0] * cum[-1]), len(cum) - 1)
    t = np.asarray(vertices, np.float64)[np.asarray(faces, np.int64)[fi]]
    r = u[:, 1:3].copy()
    flip = r.sum(axis=1) > 1.0
    r[flip] = np.abs(r[flip] - 1.0)
    e = t[:, 1:] - t[:, :1]
    return t[:, 0] + (e * r[:, :, None]).sum(axis=1), fi


def uniforms(n, seed):
    """Injected randoms for the sampler: [n, 3] in [0, 1)."""
    return np.random.default_rng(seed).random((n, 3))


# ---- box crop -------------------------------------------------------------------------------------------------------
def clip_to_box(vertices, faces, center, R, extent):
    """Triangle soup [T,3,3] f64 of mesh ∩ box, ordered by (input face, fan order).  ``R`` has the box axes as
    columns, ``extent`` the full edge lengths."""
    v = np.asarray(vertices, np.float64)
    f = np.asarray(faces, np.int64)
    c, R, half = np.asarray(center, np.float64), np.asarray(R, np.float64), 0.5 * np.asarray(extent, np.float64)
    F = len(f)
    ar = np.arange(F)
    P = np.zeros((F, 10, 3))
    P[:, :3] = v[f]
    n = np.full(F, 3)
    for pl in range(6):
        j, sg = pl >> 1, (-1.0 if pl & 1 else 1.0)
        d = half[j] - sg * ((P - c) @ R[:, j])                  # [F, 10], inside when >= 0
        Q = np.zeros_like(P)
        m = np.zeros(F, np.int64)
        for k in range(9):
            valid = k < n
            kn = np.where(k + 1 < n, k + 1, 0)
            a, b = P[:, k], P[ar, kn]
            da, db = d[:, k], d[ar, kn]
            keep = valid & (da >= 0)
            Q[ar[keep], m[keep]] = a[keep]
            m += keep
            cross = valid & ((da >= 0) != (db >= 0))
            with np.errstate(divide="ignore", invalid="ignore"):
                t = da / (da - db)
                x = a + t[:, None] * (b - a)
            Q[ar[cross], m[cross]] = x[cross]
            m += cross
        P, n = Q, m
    ntri = np.maximum(n - 2, 0)
    out = np.zeros((int(ntri.sum()), 3, 3))
    first = np.concatenate([[0], np.cumsum(ntri)[:-1]])
    for k in range(1, 8):                                       # fan triangle k of every face that has one
        sel = k + 1 < n
        idx = first[sel] + (k - 1)
        out[idx, 0] = P[sel, 0]
        out[idx, 1] = P[sel, k]
        out[idx, 2] = P[sel, k + 1]
    return out


def soup_area(soup):
    s = np.asarray(soup, np.float64)
    return float(np.linalg.norm(np.cross(s[:, 1] - s[:, 0], s[:, 2] - s[:, 0]), axis=1).sum() / 2.0)


# ---- eval_3D_*.calc_3d_metric ---------------------------------------------------------------------------------------
def calc_3d_metric(rec_vertices, rec_faces, gt_vertices, gt_faces, u_rec, u_gt, crop_to_gt_box=False):
    """[[acc], [comp], [ratio@0.01], [ratio@0.05]] with injected sampler randoms, or None when the crop is empty."""
    if crop_to_gt_box:
        from vmap_b200.mesh import oriented_bounds
        center, R, ext = oriented_bounds(np.asarray(gt_vertices, np.float64))
        soup = clip_to_box(rec_vertices, rec_faces, center, R, ext / 0.9)
        if len(soup) == 0:
            return None
        rec_vertices, rec_faces = soup.reshape(-1, 3), np.arange(3 * len(soup)).reshape(-1, 3)
    rec = sample_surface(rec_vertices, rec_faces, u_rec)[0].astype(np.float32)      # the kernel stores fp32 points
    gt = sample_surface(gt_vertices, gt_faces, u_gt)[0].astype(np.float32)
    return [[accuracy(gt, rec)], [completion(gt, rec)], [completion_ratio(gt, rec, 0.01)],
            [completion_ratio(gt, rec, 0.05)]]
