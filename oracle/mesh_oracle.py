"""CPU oracle of the meshing path (numpy): the marching-cubes triangulation table generator, a marching cubes that
uses that table with the same vertex / face order and arithmetic as the CUDA kernels, and the pinhole unprojection
of sceneObject.get_bound.

Table rule.  Cube corner c sits at (c & 1, c >> 1 & 1, c >> 2 & 1) along volume axes (0, 1, 2); edge e joins corners
(c0, c0 | 1 << a), numbered axis-major then by c0.  A corner is inside when its value exceeds the level.
  * On a cube face with two crossed edges, one segment joins them.  On a face with four (its two inside corners
    are diagonal), the contour separates the inside corners: each inside corner is cut off by the segment joining
    its two face edges.  Two cells sharing a face see the same corner values and cut it the same way, so the mesh
    has no cracks.
  * Each segment is directed so that, seen with the outward face normal n_f and the in-face direction u from the
    inside corners towards the outside ones, (u x (q - p)) . n_f < 0.  Every crossed edge then has one incoming and
    one outgoing segment, the segments chain into closed cycles, and a cycle traversed in that direction has its
    right-hand normal pointing from inside (high values) to outside.
  * Cycles are taken in order of their smallest edge index.  Each is fan-triangulated from the smallest of its
    edges whose chords all cross the cube's interior (no chord lies in a cube face, where the neighbouring cell
    could draw the same chord); every cycle of the 256 cases has such an edge.

``python -m oracle.mesh_oracle`` rewrites vmap_b200/csrc/mc_table.cuh; tests/test_mesh_oracle.py checks that the
committed header is what the generator prints.
"""
from __future__ import annotations

import os
from typing import List, Tuple

import numpy as np

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vmap_b200", "csrc", "mc_table.cuh")

CORNERS = np.array([[(c >> 0) & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)], dtype=np.float64)
EDGES: List[Tuple[int, int, int]] = [(c0, c0 | (1 << a), a) for a in range(3) for c0 in range(8) if not (c0 >> a) & 1]
FACES = [(a, s) for a in range(3) for s in (0, 1)]          # face of corners with bit a == s


def _face_segments(case: int, a: int, s: int):
    """Directed segments (edge p, edge q) that the contour of ``case`` draws on face (a, s)."""
    ins = [(case >> c) & 1 for c in range(8)]
    n_f = np.zeros(3)
    n_f[a] = 1.0 if s else -1.0
    corners = [c for c in range(8) if ((c >> a) & 1) == s]
    fedges = [e for e, (c0, c1, ax) in enumerate(EDGES) if ax != a and ((c0 >> a) & 1) == s]
    crossed = [e for e in fedges if ins[EDGES[e][0]] != ins[EDGES[e][1]]]
    mid = {e: 0.5 * (CORNERS[EDGES[e][0]] + CORNERS[EDGES[e][1]]) for e in fedges}
    segs = []
    if len(crossed) == 2:
        cin = [c for c in corners if ins[c]]
        cout = [c for c in corners if not ins[c]]
        u = CORNERS[cout].mean(0) - CORNERS[cin].mean(0)
        segs.append((crossed[0], crossed[1], u))
    elif len(crossed) == 4:                                    # diagonal: cut every inside corner off on its own
        for c in corners:
            if ins[c]:
                p, q = [e for e in fedges if c in EDGES[e][:2]]
                u = 0.5 * (mid[p] + mid[q]) - CORNERS[c]
                segs.append((p, q, u))
    out = []
    for p, q, u in segs:
        if np.dot(np.cross(u, mid[q] - mid[p]), n_f) > 0:
            p, q = q, p
        out.append((p, q))
    return out


def case_cycles(case: int) -> List[List[int]]:
    """Closed cycles of crossed edges of one cube case, in table order."""
    nxt = {}
    for a, s in FACES:
        for p, q in _face_segments(case, a, s):
            assert p not in nxt, (case, p)
            nxt[p] = q
    assert sorted(nxt) == sorted(nxt.values()), case          # one incoming and one outgoing segment per edge
    cycles, seen = [], set()
    for e0 in sorted(nxt):
        if e0 in seen:
            continue
        cyc, e = [], e0
        while e not in seen:
            seen.add(e)
            cyc.append(e)
            e = nxt[e]
        assert e == e0, case
        cycles.append(cyc)
    return cycles


def _edge_faces(e: int):
    c0, _, ax = EDGES[e]
    return {(a, (c0 >> a) & 1) for a in range(3) if a != ax}


def fan_apex(cyc: List[int]) -> int:
    """Position in ``cyc`` of the fan apex: the smallest edge whose chords all cross the cube's interior.  A chord
    between two edges of one cube face would lie in that face, where the neighbouring cell may draw the same chord,
    and the mesh edge would then belong to four triangles."""
    for e in sorted(cyc):
        r = cyc.index(e)
        c = cyc[r:] + cyc[:r]
        if all(not (_edge_faces(c[0]) & _edge_faces(c[i])) for i in range(2, len(c) - 1)):
            return r
    raise AssertionError(f"no interior fan apex for cycle {cyc}")


def make_table():
    """(ntri [256] int, tri [256][max_tri][3] int (edge indices, unused rows -1))."""
    tris = []
    for case in range(256):
        t = []
        for cyc in case_cycles(case):
            r = fan_apex(cyc)
            cyc = cyc[r:] + cyc[:r]
            t += [(cyc[0], cyc[i], cyc[i + 1]) for i in range(1, len(cyc) - 1)]
        tris.append(t)
    mt = max(len(t) for t in tris)
    ntri = np.array([len(t) for t in tris], dtype=np.int64)
    tri = -np.ones((256, mt, 3), dtype=np.int64)
    for case, t in enumerate(tris):
        if t:
            tri[case, :len(t)] = t
    return ntri, tri


def header_text() -> str:
    ntri, tri = make_table()
    mt = tri.shape[1]
    L = ["// Marching-cubes tables.  GENERATED by `python -m oracle.mesh_oracle` from the face-separation rule stated",
         "// there -- do not edit by hand (tests/test_mesh_oracle.py checks this file against the generator).",
         "// Corner c = (c&1, c>>1&1, c>>2&1) along volume axes (0,1,2); edge e = (c0, c0 | 1<<axis), see mc_edge_*.",
         "#pragma once", "",
         f"#define VMB_MC_MAX_TRI {mt}", "",
         "// edge -> (axis, lower corner)",
         "__device__ const unsigned char mc_edge_axis[12] = {" + ", ".join(str(a) for _, _, a in EDGES) + "};",
         "__device__ const unsigned char mc_edge_c0[12] = {" + ", ".join(str(c) for c, _, _ in EDGES) + "};", "",
         "// triangles per case (case bit c = corner c inside)",
         "__device__ const unsigned char mc_ntri[256] = {"]
    for r in range(0, 256, 32):
        L.append("  " + ", ".join(str(int(x)) for x in ntri[r:r + 32]) + ",")
    L += ["};", "", f"// edge triples per case, {mt} rows of 3, unused entries 255",
          f"__device__ const unsigned char mc_tri[256][{3 * mt}] = {{"]
    for case in range(256):
        row = [str(int(x)) if x >= 0 else "255" for x in tri[case].reshape(-1)]
        L.append("  {" + ", ".join(row) + "},")
    L += ["};", ""]
    return "\n".join(L)


# ---- marching cubes ---------------------------------------------------------------------------------------------------
def gradient(v: np.ndarray) -> np.ndarray:
    """[nx,ny,nz,3] fp32 central differences, one-sided at the volume border."""
    g = np.empty(v.shape + (3,), dtype=np.float32)
    for a in range(3):
        n = v.shape[a]
        sl = lambda i: tuple(slice(None) if d != a else i for d in range(3))
        ga = np.empty_like(v)
        ga[sl(slice(1, n - 1))] = (v[sl(slice(2, n))] - v[sl(slice(0, n - 2))]) * np.float32(0.5)
        ga[sl(0)] = v[sl(1)] - v[sl(0)]
        ga[sl(n - 1)] = v[sl(n - 1)] - v[sl(n - 2)]
        g[..., a] = ga
    return g


def marching_cubes(vol, level: float = 0.5, affine=None):
    """(vertices [V,3] f32, faces [F,3] int32, normals [V,3] f32) in the CUDA kernels' order: vertices by (grid point
    linear index, edge axis), faces by (cell linear index, table order).  ``affine`` [3,4]: index -> world."""
    v = np.ascontiguousarray(vol, dtype=np.float32)
    nx, ny, nz = v.shape
    lv = np.float32(level)
    M = np.eye(3) if affine is None else np.asarray(affine, np.float64)[:, :3]
    off = np.zeros(3) if affine is None else np.asarray(affine, np.float64)[:, 3]
    ins = v > lv
    ntri, tri = make_table()
    crossed = np.zeros(v.shape + (3,), dtype=bool)
    crossed[:-1, :, :, 0] = ins[:-1] != ins[1:]
    crossed[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    crossed[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    cflat = crossed.reshape(-1, 3)
    cnt = cflat.sum(1)
    base = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
    below = np.stack([np.zeros(len(cnt), np.int64), cflat[:, 0], cflat[:, 0].astype(np.int64) + cflat[:, 1]], 1)
    pt, ax = np.nonzero(cflat)                                   # point-major, axis-minor
    idx = np.stack(np.unravel_index(pt, v.shape), 1)
    vflat = v.reshape(-1)
    step = np.array([ny * nz, nz, 1])[ax]
    va, vb = vflat[pt], vflat[pt + step]
    t = (lv - va) / (vb - va)
    pos = idx.astype(np.float32)
    pos[np.arange(len(pt)), ax] += t
    g = gradient(v).reshape(-1, 3)
    ga, gb = g[pt], g[pt + step]
    nrm = -(ga + t[:, None] * (gb - ga))
    nrm = (nrm.astype(np.float64) @ np.linalg.inv(M)).astype(np.float32)      # inverse transpose: n' = M^-T n
    ln = np.sqrt((nrm.astype(np.float64) ** 2).sum(1))
    nrm = np.where(ln[:, None] > 0, nrm / np.where(ln > 0, ln, 1)[:, None], 0).astype(np.float32)
    verts = (pos.astype(np.float64) @ M.T + off).astype(np.float32)
    # cells
    case = np.zeros((nx - 1, ny - 1, nz - 1), dtype=np.int64)
    for c in range(8):
        i, j, k = (c >> 0) & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= ins[i:nx - 1 + i, j:ny - 1 + j, k:nz - 1 + k].astype(np.int64) << c
    cf = case.reshape(-1)
    cells = np.nonzero(ntri[cf])[0]
    faces = []
    if len(cells):
        cidx = np.stack(np.unravel_index(cells, case.shape), 1)
        mt = tri.shape[1]
        rows = tri[cf[cells]].reshape(len(cells), mt * 3)            # [C, mt*3] edge ids (-1 unused)
        valid = rows >= 0
        e = np.where(valid, rows, 0)
        c0 = np.array([c for c, _, _ in EDGES])[e]
        a = np.array([x for _, _, x in EDGES])[e]
        q = cidx[:, None, :] + CORNERS[c0].astype(np.int64)
        ql = (q[..., 0] * ny + q[..., 1]) * nz + q[..., 2]
        vid = base[ql] + below[ql, a]
        faces = vid[valid].reshape(-1, 3)
    faces = np.asarray(faces, dtype=np.int32).reshape(-1, 3)
    return verts, faces, nrm


# ---- unprojection (open3d pinhole model, PointCloud.create_from_depth_image) ---------------------------------------
def unproject(depth, select, t_wc, fx, fy, cx, cy):
    """World points [n,3] f64 of the selected pixels with depth > 0, in (keyframe, u, v) order.
    ``depth`` / ``select`` [KF,W,H] (u indexes W, v indexes H), ``t_wc`` [KF,4,4]."""
    out = []
    for kf in range(depth.shape[0]):
        d = np.asarray(depth[kf], np.float64)
        u, vv = np.nonzero(np.asarray(select[kf], bool) & (d > 0))
        z = d[u, vv]
        pc = np.stack([(u - cx) * z / fx, (vv - cy) * z / fy, z], 1)
        T = np.asarray(t_wc[kf], np.float64)
        out.append(pc @ T[:3, :3].T + T[:3, 3])
    return np.concatenate(out, 0) if out else np.zeros((0, 3))


# ---- mesh checks used by the tests ----------------------------------------------------------------------------------
def directed_edge_check(faces) -> bool:
    """Every edge shared by exactly two faces with opposite directions (closed, consistently wound)."""
    f = np.asarray(faces, np.int64)
    if len(f) == 0:
        return True
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 0)
    key = d[:, 0] * (int(d.max()) + 1) + d[:, 1]
    rkey = d[:, 1] * (int(d.max()) + 1) + d[:, 0]
    if len(np.unique(key)) != len(key):                        # a directed edge used twice
        return False
    return bool(np.isin(rkey, key).all())


def euler_characteristic(verts, faces) -> int:
    f = np.asarray(faces, np.int64)
    d = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 0), 1)
    n_e = len(np.unique(d[:, 0] * (int(d.max()) + 1) + d[:, 1]))
    n_v = len(np.unique(f))
    return n_v - n_e + len(f)


def signed_volume(verts, faces) -> float:
    p = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return float(np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0)


if __name__ == "__main__":
    with open(HEADER, "w") as f:
        f.write(header_text())
    print("wrote", HEADER)
