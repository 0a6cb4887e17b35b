"""numpy / scipy restatement of the open3d 0.16 pieces that the reference's ScanNet path uses (utils.py:112-264,
dataset.py:177-184).  It can be put in ``sys.modules['open3d']`` so that the reference's own dataset.ScanNet and
utils.box_filter run without open3d.

TEST INFRASTRUCTURE ONLY, and RESTATED, NOT CHECKED: open3d cannot be installed where this project is developed, so
nothing here was run side by side with open3d (the same standing trimesh has in INTEGRATION.md section 5).  Each
routine follows open3d 0.16's C++ source, with the arithmetic order spelled out where open3d leaves it to Eigen:

* ``PointCloud.create_from_depth_image`` (float depth): ``depth_scale`` / ``depth_trunc`` are ignored for a float
  image; pixels with z > 0 are kept in row-major (v, u) order; x = (u - cx) * z / fx, y = (v - cy) * z / fy in fp64;
  point = camera_pose . [x, y, z, 1] with camera_pose = inv(extrinsic), each row summed left to right.
* ``voxel_down_sample``: min_bound = min(points) - 0.5 * voxel, key = floor((p - min_bound) / voxel), each output
  point the mean of its voxel's points summed in input order.  open3d emits an unordered_map's order; here the
  output is in ascending (kx, ky, kz) order.
* ``OrientedBoundingBox.create_from_points``: qhull vertices, raw-moment mean / covariance, eigenvectors sorted by
  descending eigenvalue with open3d's three swaps, R[:, 2] = R[:, 0] x R[:, 1], AABB in that frame.  A qhull
  failure raises RuntimeError as open3d does.
* ``get_point_indices_within_bounding_box``: the inclusive test |d . dx| <= dx . dx on the three half axes.
"""
from __future__ import annotations

import sys
import types

import numpy as np
from scipy.spatial import ConvexHull, QhullError


def _as_points(p):
    return np.asarray(p, dtype=np.float64).reshape(-1, 3)


def dot3(a, b):
    """a . b per row, summed left to right with no fused multiply-add."""
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


class PinholeCameraIntrinsic:
    def __init__(self, width=-1, height=-1, fx=0.0, fy=0.0, cx=0.0, cy=0.0):
        self.width, self.height = int(width), int(height)
        self.intrinsic_matrix = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], np.float64)

    def get_focal_length(self):
        return float(self.intrinsic_matrix[0, 0]), float(self.intrinsic_matrix[1, 1])

    def get_principal_point(self):
        return float(self.intrinsic_matrix[0, 2]), float(self.intrinsic_matrix[1, 2])


class Image:
    def __init__(self, data):
        self.data = np.asarray(data)


def unproject(depth, fx, fy, cx, cy, camera_pose):
    """Float-depth unprojection of every z > 0 pixel of an [H, W] image, row-major, fp64, no FMA."""
    depth = np.asarray(depth)
    v, u = np.nonzero(depth > 0)
    z = depth[v, u].astype(np.float64)
    x = (u.astype(np.float64) - cx) * z / fx
    y = (v.astype(np.float64) - cy) * z / fy
    P = np.asarray(camera_pose, np.float64)
    out = np.empty((len(z), 3), np.float64)
    for r in range(3):
        out[:, r] = P[r, 0] * x + P[r, 1] * y + P[r, 2] * z + P[r, 3]
    return out


def voxel_down_sample(points, voxel_size):
    """open3d 0.16 VoxelDownSample, output in ascending voxel-key order."""
    p = _as_points(points)
    if len(p) == 0:
        return p.copy()
    vs = float(voxel_size)
    min_bound = p.min(axis=0) - vs * 0.5
    key = np.floor((p - min_bound) / vs).astype(np.int64)
    order = np.lexsort((key[:, 2], key[:, 1], key[:, 0]))           # stable: input order inside a voxel
    ks = key[order]
    first = np.ones(len(ks), bool)
    first[1:] = np.any(ks[1:] != ks[:-1], axis=1)
    group = np.cumsum(first) - 1
    n_out = int(group[-1]) + 1
    acc = np.zeros((n_out, 3), np.float64)
    np.add.at(acc, group, p[order])                                # sequential, in input order
    cnt = np.bincount(group, minlength=n_out).astype(np.float64)
    return acc / cnt[:, None]


def obb_from_points(points):
    """open3d 0.16 OrientedBoundingBox::CreateFromPoints -> (center, R, extent); RuntimeError on a qhull failure."""
    p = _as_points(points)
    try:
        hull = ConvexHull(p)
    except (QhullError, ValueError) as e:
        raise RuntimeError(f"QH6214 qhull: {e}") from None
    hv = p[hull.vertices]
    n = float(len(hv))
    m = hv.sum(axis=0) / n
    xx = np.stack([hv[:, 0] * hv[:, 0], hv[:, 0] * hv[:, 1], hv[:, 0] * hv[:, 2],
                   hv[:, 1] * hv[:, 1], hv[:, 1] * hv[:, 2], hv[:, 2] * hv[:, 2]], axis=1).sum(axis=0) / n
    cov = np.array([[xx[0] - m[0] * m[0], xx[1] - m[0] * m[1], xx[2] - m[0] * m[2]],
                    [0.0, xx[3] - m[1] * m[1], xx[4] - m[1] * m[2]],
                    [0.0, 0.0, xx[5] - m[2] * m[2]]])
    cov[1, 0], cov[2, 0], cov[2, 1] = cov[0, 1], cov[0, 2], cov[1, 2]
    evals, R = np.linalg.eigh(cov)
    evals, R = evals.copy(), R.copy()
    for a, b in ((1, 0), (2, 0), (2, 1)):                          # open3d's three swaps -> descending
        if evals[a] > evals[b]:
            evals[[a, b]] = evals[[b, a]]
            R[:, [a, b]] = R[:, [b, a]]
    R[:, 0] /= np.sqrt(dot3(R[:, 0], R[:, 0]))
    R[:, 1] /= np.sqrt(dot3(R[:, 1], R[:, 1]))
    R[:, 2] = np.cross(R[:, 0], R[:, 1])
    d = hv - m
    local = np.stack([dot3(d, R[:, j]) for j in range(3)], axis=1)
    lo, hi = local.min(axis=0), local.max(axis=0)
    c_loc = (lo + hi) * 0.5
    center = np.array([dot3(R[r], c_loc) for r in range(3)]) + m
    return center, R, hi - lo


def box_axes(center, R, extent):
    """The half axes dx, dy, dz and their squared lengths used by the inside test."""
    R = np.asarray(R, np.float64)
    ext = np.asarray(extent, np.float64)
    ax = [R[:, j] * (0.5 * ext[j]) for j in range(3)]
    return np.asarray(center, np.float64), ax, [dot3(a, a) for a in ax]


def inside_box(points, center, R, extent):
    """Inclusive oriented-box test of open3d 0.16 GetPointIndicesWithinBoundingBox, as a boolean mask."""
    c, ax, nn = box_axes(center, R, extent)
    d = _as_points(points) - c
    ok = np.ones(len(d), bool)
    for a, n in zip(ax, nn):
        ok &= np.abs(dot3(d, a)) <= n
    return ok


class PointCloud:
    def __init__(self, points=None):
        self.points = _as_points(points if points is not None else np.zeros((0, 3)))

    @staticmethod
    def create_from_depth_image(depth, intrinsic, extrinsic=np.eye(4), depth_scale=1000.0, depth_trunc=1000.0,
                                stride=1, project_valid_depth_only=True):
        d = depth.data if isinstance(depth, Image) else np.asarray(depth)
        if d.dtype != np.float32 or stride != 1 or not project_valid_depth_only:
            raise NotImplementedError("stand-in covers float depth, stride 1, valid pixels only")
        fx, fy = intrinsic.get_focal_length()
        cx, cy = intrinsic.get_principal_point()
        return PointCloud(unproject(d, fx, fy, cx, cy, np.linalg.inv(np.asarray(extrinsic, np.float64))))

    def __add__(self, other):
        return PointCloud(np.concatenate([self.points, other.points]))

    def __iadd__(self, other):
        self.points = np.concatenate([self.points, other.points])
        return self

    def select_by_index(self, indices, invert=False):
        idx = np.asarray(indices, np.int64)
        if invert:
            keep = np.ones(len(self.points), bool)
            keep[idx] = False
            return PointCloud(self.points[keep])
        return PointCloud(self.points[idx])

    def voxel_down_sample(self, voxel_size):
        return PointCloud(voxel_down_sample(self.points, voxel_size))


class OrientedBoundingBox:
    def __init__(self, center=np.zeros(3), R=np.eye(3), extent=np.zeros(3)):
        self.center = np.asarray(center, np.float64).copy()
        self.R = np.asarray(R, np.float64).copy()
        self.extent = np.asarray(extent, np.float64).copy()

    @staticmethod
    def create_from_points(points, robust=False):
        return OrientedBoundingBox(*obb_from_points(points))

    def get_center(self):
        return self.center.copy()

    def scale(self, scale, center):
        self.extent = scale * self.extent
        self.center = scale * (self.center - np.asarray(center, np.float64)) + np.asarray(center, np.float64)
        return self

    def get_point_indices_within_bounding_box(self, points):
        return list(np.nonzero(inside_box(points, self.center, self.R, self.extent))[0])


def as_module() -> types.ModuleType:
    """A module object that can stand in for ``open3d`` (camera, geometry, utility)."""
    m = types.ModuleType("open3d")
    m.camera = types.SimpleNamespace(PinholeCameraIntrinsic=PinholeCameraIntrinsic)
    m.geometry = types.SimpleNamespace(PointCloud=PointCloud, Image=Image, OrientedBoundingBox=OrientedBoundingBox)
    m.utility = types.SimpleNamespace(Vector3dVector=_as_points)
    m.__standin__ = True
    return m


def install():
    """Put the stand-in in sys.modules['open3d'] (replacing whatever is there); returns the previous entry."""
    prev = sys.modules.get("open3d")
    sys.modules["open3d"] = as_module()
    return prev
