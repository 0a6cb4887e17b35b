// K8: exact segmented 3-D convex hull and the minimum-volume oriented box fitted to it, for sceneObject.get_bound and
// the per-object metric's GT box.
//
// Predicate: orient(a, b, c, p) = sign det[a - p; b - p; c - p], decided exactly.  The fp64 determinant is taken when
// it clears Shewchuk's static bound ((7 + 56 eps) eps times the permanent); otherwise the determinant of the exact
// differences is evaluated in expansion arithmetic (two-sum / two-product, zero-eliminating grow and scale).
// A facet (a, b, c) is stored with its outward normal along (b - a) x (c - a): p is strictly above it iff
// orient(a, b, c, p) < 0.
//
// Hull of one point list (one CTA): incremental with strict visibility.  The first simplex is the first four affinely
// independent points of (26 seeds, then the list in input order); the seeds are the argmax / argmin along 13 fixed
// directions, ties to the lowest position, so a value's lowest index is always inserted before its copies and a copy
// of an inserted point is never strictly above a facet.  Each chunk of 256 points is first tested against the
// current hull in parallel; the survivors are inserted in input order: a parallel scan marks the strictly visible
// facets, one thread replaces them by the cone from the horizon (visible list sorted, so slots are deterministic).
// Facets live in handle scratch (vertices, neighbours across edge (v_j, v_j+1), state) with a free list; a hull of
// m points never holds more than 2m - 4 facets.  Afterwards a triangulation vertex is an extreme point iff its
// incident facets lie in at least three distinct planes (one plane: inside a face; two: on an edge), decided with
// the exact predicate.  Every extreme point is a triangulation vertex, so this is the exact extreme-point set.
//
// Hull of hulls: every set with more than TILE points is cut into tiles of TILE consecutive points (one CTA each);
// a tile keeps its extreme points (all of them when it is flat), the survivors are compacted in (set, input order)
// and the pass repeats, up to ROUNDS times, while a set still has more than TILE points and shrinks.  A non-vertex
// of a subset is never a vertex of the whole set.  The last pass runs one CTA per set and emits the facets.
// Nothing waits for the host: set sizes are read and scanned on the device.
//
// Box (trimesh.bounds.oriented_bounds as vmap_b200/mesh.py restates it): unit facet normals rounded to 1e-10 (rint
// of x * 1e10, / 1e10, as np.round), one candidate per distinct rounded normal.  Per candidate (one CTA): b1 =
// normalise(n x (|n0| < 0.9 ? e0 : e1)), b2 = n x b1, the height along n over the hull vertices, and the minimum-area
// rectangle of the projected vertices over the directions of the silhouette edges (hull edges whose facets' unit
// normals have dot products with n of opposite sign, or within 1e-9 of zero: a superset of the 2-D hull's edge
// directions).  The least volume wins, exact ties to the lexicographically smallest rounded normal (np.unique's
// order); R = [a0 a1 n] with the normal axis flipped when det R < 0.
#pragma once
#include "common.cuh"
#include <limits.h>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

namespace hull {

constexpr int NT = 256;
constexpr int TILE = 4096;
constexpr int ROUNDS = 5;
constexpr int NDIR = 13;
enum { ST_OK = 0, ST_TOO_FEW = 1, ST_FLAT = 2, ST_BAD = 3 };   // VMB_HULL_* in the header
enum { DEAD = 0, ALIVE = 1, VIS = 2 };

// ---- exact orientation ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void two_sum(double a, double b, double& x, double& y) {
  x = __dadd_rn(a, b);
  const double bv = __dsub_rn(x, a), av = __dsub_rn(x, bv);
  y = __dadd_rn(__dsub_rn(a, av), __dsub_rn(b, bv));
}
__device__ __forceinline__ void two_diff(double a, double b, double& x, double& y) {
  x = __dsub_rn(a, b);
  const double bv = __dsub_rn(a, x), av = __dadd_rn(x, bv);
  y = __dadd_rn(__dsub_rn(a, av), __dsub_rn(bv, b));
}
__device__ __forceinline__ void two_prod(double a, double b, double& x, double& y) {
  x = __dmul_rn(a, b);
  y = fma(a, b, -x);
}
// h = e + b (e nonoverlapping, increasing magnitude); h may alias e.
__device__ __forceinline__ int grow_exp(int elen, const double* e, double b, double* h) {
  double Q = b;
  int hi = 0;
  for (int i = 0; i < elen; ++i) {
    double Qn, hh;
    two_sum(Q, e[i], Qn, hh);
    Q = Qn;
    if (hh != 0.0) h[hi++] = hh;
  }
  if (Q != 0.0 || hi == 0) h[hi++] = Q;
  return hi;
}
// h = e * b; h must not alias e.
__device__ __forceinline__ int scale_exp(int elen, const double* e, double b, double* h) {
  double Q, hh;
  two_prod(e[0], b, Q, hh);
  int hi = 0;
  if (hh != 0.0) h[hi++] = hh;
  for (int i = 1; i < elen; ++i) {
    double p1, p0, s;
    two_prod(e[i], b, p1, p0);
    two_sum(Q, p0, s, hh);
    if (hh != 0.0) h[hi++] = hh;
    two_sum(p1, s, Q, hh);
    if (hh != 0.0) h[hi++] = hh;
  }
  if (Q != 0.0 || hi == 0) h[hi++] = Q;
  return hi;
}
// h += e * f, with tmp of at least 2 * elen entries.
__device__ __forceinline__ int madd_exp(int hlen, double* h, int elen, const double* e, int flen, const double* f,
                                        double* tmp, double sign) {
  for (int i = 0; i < flen; ++i) {
    const int tl = scale_exp(elen, e, sign * f[i], tmp);
    for (int k = 0; k < tl; ++k) hlen = grow_exp(hlen, h, tmp[k], h);
  }
  return hlen;
}

// sign det[a - p; b - p; c - p] in expansion arithmetic (exact differences, exact products and sums).
__device__ __noinline__ int orient_exact(double3 a, double3 b, double3 c, double3 p) {
  double r[3][3][2];
  int rl[3][3];
  const double ra[3][3] = {{a.x, a.y, a.z}, {b.x, b.y, b.z}, {c.x, c.y, c.z}}, pp[3] = {p.x, p.y, p.z};
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) {
      double hi, lo;
      two_diff(ra[i][k], pp[k], hi, lo);
      if (lo != 0.0) { r[i][k][0] = lo; r[i][k][1] = hi; rl[i][k] = 2; }
      else { r[i][k][0] = hi; rl[i][k] = 1; }
    }
  double m[16], prod[8], tmp[32], t[64], det[192];
  int dl = 1;
  det[0] = 0.0;
  // det = sum_k r0[k] * (r1[k1] r2[k2] - r1[k2] r2[k1]), (k, k1, k2) cyclic
  for (int k = 0; k < 3; ++k) {
    const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
    int ml = 1;
    m[0] = 0.0;
    int pl = 1;
    prod[0] = 0.0;
    pl = madd_exp(pl, prod, rl[1][k1], r[1][k1], rl[2][k2], r[2][k2], tmp, 1.0);
    for (int i = 0; i < pl; ++i) ml = grow_exp(ml, m, prod[i], m);
    pl = 1;
    prod[0] = 0.0;
    pl = madd_exp(pl, prod, rl[1][k2], r[1][k2], rl[2][k1], r[2][k1], tmp, -1.0);
    for (int i = 0; i < pl; ++i) ml = grow_exp(ml, m, prod[i], m);
    int tl = 1;
    t[0] = 0.0;
    tl = madd_exp(tl, t, ml, m, rl[0][k], r[0][k], tmp, 1.0);
    for (int i = 0; i < tl; ++i) dl = grow_exp(dl, det, t[i], det);
  }
  const double s = det[dl - 1];
  return (s > 0.0) - (s < 0.0);
}

__device__ __forceinline__ int orient(double3 a, double3 b, double3 c, double3 p) {
  const double adx = a.x - p.x, bdx = b.x - p.x, cdx = c.x - p.x;
  const double ady = a.y - p.y, bdy = b.y - p.y, cdy = c.y - p.y;
  const double adz = a.z - p.z, bdz = b.z - p.z, cdz = c.z - p.z;
  const double bc = __dmul_rn(bdx, cdy), cb = __dmul_rn(cdx, bdy);
  const double ca = __dmul_rn(cdx, ady), ac = __dmul_rn(adx, cdy);
  const double ab = __dmul_rn(adx, bdy), ba = __dmul_rn(bdx, ady);
  const double det = __dadd_rn(__dadd_rn(__dmul_rn(adz, __dsub_rn(bc, cb)), __dmul_rn(bdz, __dsub_rn(ca, ac))),
                               __dmul_rn(cdz, __dsub_rn(ab, ba)));
  const double perm = __dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn(fabs(bc), fabs(cb)), fabs(adz)),
                                          __dmul_rn(__dadd_rn(fabs(ca), fabs(ac)), fabs(bdz))),
                                __dmul_rn(__dadd_rn(fabs(ab), fabs(ba)), fabs(cdz)));
  const double eps = 1.1102230246251565e-16;
  const double bound = (7.0 + 56.0 * eps) * eps * perm;
  if (det > bound) return 1;
  if (-det > bound) return -1;
  return orient_exact(a, b, c, p);
}

__device__ __forceinline__ double3 ld(const double* P, int g) {
  return make_double3(P[3 * (size_t)g], P[3 * (size_t)g + 1], P[3 * (size_t)g + 2]);
}
__device__ __forceinline__ bool above(const double* P, const int* v, double3 p) {
  return orient(ld(P, v[0]), ld(P, v[1]), ld(P, v[2]), p) < 0;
}

// ---- parameters, scratch --------------------------------------------------------------------------------------------
struct Params {
  const double* pts; long long n;                 // [n][3]
  const int* set_size; int size_stride; int n_sets;
  unsigned char* is_vertex; int* vertex_count; int* status;
  int* facets; int* facet_nbr; int* facet_count;  // facets of set s at rows 2 * start[s] + [0, facet_count[s])
  // scratch
  int* size;           // [n_sets] sizes clamped to >= 0
  int* start;          // [n_sets + 1] exclusive scan of size
  int* cnt[3];         // [n_sets + 1] survivors per set (the scan needs one more entry); rounds rotate over three
  int* off[2];         // [n_sets + 1] first list position of each set
  int* list[2];        // [n] survivor point indices in (set, input order)
  int* red;            // [n_sets] the set is cut into tiles this round
  int* ntile;          // [n_sets + 1]
  int* tile_start;     // [n_sets + 1]
  unsigned char* mark; // [n] tile survivors by point index
  unsigned char* keep; // [n] tile survivors by list position
  int* n_sel;          // [1]
  int* start_at; int* end_at;   // [n] per point index
  int* fv; int* fn; int* fs; int* vis; int* fre; int* hz;  // facet work regions, capacity fcap (hz: 3 per slot)
  long long fcap;
};

__host__ __device__ inline long long max_tiles(long long n, int n_sets) { return n / TILE + n_sets + 1; }
__host__ __device__ inline long long facet_cap(long long n, int n_sets) { return 2 * n + 8 * (max_tiles(n, n_sets) + 1); }

struct Work {
  int* fv; int* fn; int* fs; int* vis; int* fre; int* hz;
};
__device__ __forceinline__ Work work_at(const Params& q, long long base) {
  return Work{q.fv + 3 * base, q.fn + 3 * base, q.fs + base, q.vis + base, q.fre + base, q.hz + 3 * base};
}

struct Smem {
  int hw, nfree, nvis, pick, nseed, nf, nvert;
  int cand[NT];
  int seed[2 * NDIR];
  double wv[NT / 32][2 * NDIR];
  int wi[NT / 32][2 * NDIR];
};

__device__ __forceinline__ bool same_pt(double3 a, double3 b) { return a.x == b.x && a.y == b.y && a.z == b.z; }

__device__ __forceinline__ bool collinear(double3 a, double3 b, double3 p) {
  // orient(a, b, p, a + delta e_k) = +-delta (b - a) x (p - a) . e_k, delta != 0 exactly
  const double3 r0 = make_double3(a.x != 0.0 ? 2.0 * a.x : 1.0, a.y, a.z);
  const double3 r1 = make_double3(a.x, a.y != 0.0 ? 2.0 * a.y : 1.0, a.z);
  const double3 r2 = make_double3(a.x, a.y, a.z != 0.0 ? 2.0 * a.z : 1.0);
  return orient(a, b, p, r0) == 0 && orient(a, b, p, r1) == 0 && orient(a, b, p, r2) == 0;
}

// Candidate test k against the points chosen so far: 1 differs from s0, 2 not collinear with s0 s1, 3 off the plane.
__device__ __forceinline__ bool simplex_ok(int k, double3 p, const double3* s) {
  if (k == 1) return !same_pt(p, s[0]);
  if (k == 2) return !collinear(s[0], s[1], p);
  return orient(s[0], s[1], s[2], p) != 0;
}

// Position (in the list) of the first point of (seeds, list) passing simplex_ok(k), or -1.
__device__ int first_ok(const double* P, const int* ids, int m, int k, const double3* s, Smem& sm) {
  if (threadIdx.x == 0) {
    sm.pick = INT_MAX;
    for (int i = 0; i < sm.nseed; ++i)
      if (simplex_ok(k, ld(P, ids[sm.seed[i]]), s)) { sm.pick = -1 - sm.seed[i]; break; }
  }
  __syncthreads();
  if (sm.pick == INT_MAX)
    for (int i = threadIdx.x; i < m; i += NT)
      if (i < sm.pick && simplex_ok(k, ld(P, ids[i]), s)) atomicMin(&sm.pick, i);
  __syncthreads();
  const int r = sm.pick;
  __syncthreads();
  return r == INT_MAX ? -1 : (r < 0 ? -1 - r : r);
}

// The 26 seeds: argmax / argmin of 13 integer directions, ties to the lowest position.
__device__ void find_seeds(const double* P, const int* ids, int m, Smem& sm) {
  const int D[NDIR][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {1, 1, 0}, {1, -1, 0}, {1, 0, 1}, {1, 0, -1},
                          {0, 1, 1}, {0, 1, -1}, {1, 1, 1}, {1, 1, -1}, {1, -1, 1}, {-1, 1, 1}};
  double bv[2 * NDIR];
  int bi[2 * NDIR];
#pragma unroll
  for (int d = 0; d < 2 * NDIR; ++d) { bv[d] = -INFINITY; bi[d] = INT_MAX; }
  for (int i = threadIdx.x; i < m; i += NT) {
    const double3 p = ld(P, ids[i]);
#pragma unroll
    for (int d = 0; d < NDIR; ++d) {
      const double v = D[d][0] * p.x + D[d][1] * p.y + D[d][2] * p.z;
      if (v > bv[2 * d]) { bv[2 * d] = v; bi[2 * d] = i; }
      if (-v > bv[2 * d + 1]) { bv[2 * d + 1] = -v; bi[2 * d + 1] = i; }
    }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int d = 0; d < 2 * NDIR; ++d) {
    double v = bv[d];
    int i = bi[d];
    for (int o = 16; o > 0; o >>= 1) {
      const double v2 = __shfl_xor_sync(0xffffffffu, v, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
      if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
    }
    if (lane == 0) { sm.wv[w][d] = v; sm.wi[w][d] = i; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int ns = 0;
    for (int d = 0; d < 2 * NDIR; ++d) {
      double v = sm.wv[0][d];
      int i = sm.wi[0][d];
      for (int k = 1; k < NT / 32; ++k)
        if (sm.wv[k][d] > v || (sm.wv[k][d] == v && sm.wi[k][d] < i)) { v = sm.wv[k][d]; i = sm.wi[k][d]; }
      if (i == INT_MAX) continue;
      bool dup = false;
      for (int k = 0; k < ns; ++k) dup |= sm.seed[k] == i;
      if (!dup) sm.seed[ns++] = i;
    }
    sm.nseed = ns;
  }
  __syncthreads();
}

// Inserts point g: replaces the facets it is strictly above by the cone from their horizon.
__device__ void insert_point(const double* P, int g, const Work& w, Smem& sm, int* start_at, int* end_at) {
  const double3 p = ld(P, g);
  const int hw = sm.hw;
  for (int f = threadIdx.x; f < hw; f += NT)
    if (w.fs[f] == ALIVE && above(P, w.fv + 3 * f, p)) {
      w.fs[f] = VIS;
      w.vis[atomicAdd(&sm.nvis, 1)] = f;
    }
  __syncthreads();
  const int nv = sm.nvis;
  __syncthreads();
  if (nv == 0) return;
  if (threadIdx.x == 0) {
    int* vis = w.vis;
    for (int i = 1; i < nv; ++i) {                           // slot order: deterministic output
      const int x = vis[i];
      int j = i - 1;
      while (j >= 0 && vis[j] > x) { vis[j + 1] = vis[j]; --j; }
      vis[j + 1] = x;
    }
    int nh = 0;
    for (int i = 0; i < nv; ++i) {
      const int f = vis[i];
      for (int j = 0; j < 3; ++j) {
        const int o = w.fn[3 * f + j];
        if (w.fs[o] != VIS) {
          w.hz[3 * nh] = w.fv[3 * f + j];
          w.hz[3 * nh + 1] = w.fv[3 * f + (j + 1) % 3];
          w.hz[3 * nh + 2] = o;
          ++nh;
        }
      }
    }
    for (int i = 0; i < nv; ++i) {
      w.fs[vis[i]] = DEAD;
      w.fre[sm.nfree++] = vis[i];
    }
    for (int i = 0; i < nh; ++i) {
      const int s = sm.nfree ? w.fre[--sm.nfree] : sm.hw++;
      const int a = w.hz[3 * i], b = w.hz[3 * i + 1], o = w.hz[3 * i + 2];
      w.fv[3 * s] = a; w.fv[3 * s + 1] = b; w.fv[3 * s + 2] = g;
      w.fs[s] = ALIVE;
      w.fn[3 * s] = o;
      start_at[a] = s;
      end_at[b] = s;
      for (int k = 0; k < 3; ++k)
        if (w.fv[3 * o + k] == b && w.fv[3 * o + (k + 1) % 3] == a) w.fn[3 * o + k] = s;
      vis[i] = s;
    }
    for (int i = 0; i < nh; ++i) {
      const int s = vis[i];
      w.fn[3 * s + 1] = start_at[w.fv[3 * s + 1]];
      w.fn[3 * s + 2] = end_at[w.fv[3 * s]];
    }
    sm.nvis = 0;
  }
  __syncthreads();
}

// Is triangulation vertex v (incident to facet f0) an extreme point: do its incident facets span >= 3 planes?
__device__ bool extreme_at(const double* P, const Work& w, int v, int f0, int hw) {
  const double3 a = ld(P, w.fv[3 * f0]), b = ld(P, w.fv[3 * f0 + 1]), c = ld(P, w.fv[3 * f0 + 2]);
  int f2 = -1;
  double3 a2, b2, c2;
  int f = f0;
  for (int guard = 0; guard <= hw; ++guard) {
    int j = 0;
    while (j < 2 && w.fv[3 * f + j] != v) ++j;
    const double3 x = ld(P, w.fv[3 * f + (j + 1) % 3]), y = ld(P, w.fv[3 * f + (j + 2) % 3]);
    if (orient(a, b, c, x) != 0 || orient(a, b, c, y) != 0) {
      if (f2 < 0) {
        f2 = f;
        a2 = ld(P, w.fv[3 * f]); b2 = ld(P, w.fv[3 * f + 1]); c2 = ld(P, w.fv[3 * f + 2]);
      } else if (orient(a2, b2, c2, x) != 0 || orient(a2, b2, c2, y) != 0) {
        return true;
      }
    }
    f = w.fn[3 * f + j];
    if (f == f0) break;
  }
  return false;
}

// Hull of the m points ids[0..m) (point indices, input order), m >= 4.  Returns ST_OK or ST_FLAT; on ST_OK the
// facet structure in w (slots [0, sm.hw)) is the hull and flag(point index) has been called for every extreme point.
template <class Flag>
__device__ int hull_list(const double* P, const int* ids, int m, const Work& w, Smem& sm, int* start_at, int* end_at,
                         Flag flag) {
  find_seeds(P, ids, m, sm);
  double3 s[3];
  int pos[4];
  pos[0] = sm.seed[0];
  s[0] = ld(P, ids[pos[0]]);
  for (int k = 1; k < 4; ++k) {
    pos[k] = first_ok(P, ids, m, k, s, sm);
    if (pos[k] < 0) return ST_FLAT;
    if (k < 3) s[k] = ld(P, ids[pos[k]]);
  }
  if (threadIdx.x == 0) {
    const int g[4] = {ids[pos[0]], ids[pos[1]], ids[pos[2]], ids[pos[3]]};
    const int T[4][4] = {{0, 1, 2, 3}, {0, 3, 1, 2}, {1, 3, 2, 0}, {2, 3, 0, 1}};   // facet, then opposite vertex
    for (int f = 0; f < 4; ++f) {
      int v0 = g[T[f][0]], v1 = g[T[f][1]], v2 = g[T[f][2]];
      if (orient(ld(P, v0), ld(P, v1), ld(P, v2), ld(P, g[T[f][3]])) < 0) { const int t = v1; v1 = v2; v2 = t; }
      w.fv[3 * f] = v0; w.fv[3 * f + 1] = v1; w.fv[3 * f + 2] = v2;
      w.fs[f] = ALIVE;
    }
    for (int f = 0; f < 4; ++f)
      for (int j = 0; j < 3; ++j) {
        const int a = w.fv[3 * f + j], b = w.fv[3 * f + (j + 1) % 3];
        for (int o = 0; o < 4; ++o)
          for (int k = 0; k < 3; ++k)
            if (o != f && w.fv[3 * o + k] == b && w.fv[3 * o + (k + 1) % 3] == a) w.fn[3 * f + j] = o;
      }
    sm.hw = 4;
    sm.nfree = 0;
    sm.nvis = 0;
  }
  __syncthreads();
  for (int i = 0; i < sm.nseed; ++i) insert_point(P, ids[sm.seed[i]], w, sm, start_at, end_at);
  for (int c0 = 0; c0 < m; c0 += NT) {
    const int i = c0 + threadIdx.x;
    int out = 0;
    if (i < m) {
      const double3 p = ld(P, ids[i]);
      const int hw = sm.hw;
      for (int f = 0; f < hw && !out; ++f) out = w.fs[f] == ALIVE && above(P, w.fv + 3 * f, p);
    }
    sm.cand[threadIdx.x] = out;
    __syncthreads();
    const int lim = min(NT, m - c0);
    for (int k = 0; k < lim; ++k)
      if (sm.cand[k]) insert_point(P, ids[c0 + k], w, sm, start_at, end_at);
    __syncthreads();
  }
  // extreme points: one canonical incident facet per triangulation vertex (the largest slot)
  for (int i = threadIdx.x; i < m; i += NT) end_at[ids[i]] = -1;
  __syncthreads();
  const int hw = sm.hw;
  for (int f = threadIdx.x; f < hw; f += NT)
    if (w.fs[f] == ALIVE)
      for (int j = 0; j < 3; ++j) atomicMax(&end_at[w.fv[3 * f + j]], f);
  __syncthreads();
  for (int f = threadIdx.x; f < hw; f += NT)
    if (w.fs[f] == ALIVE)
      for (int j = 0; j < 3; ++j) {
        const int v = w.fv[3 * f + j];
        if (end_at[v] == f && extreme_at(P, w, v, f, hw)) flag(v);
      }
  __syncthreads();
  return ST_OK;
}

// ---- kernels --------------------------------------------------------------------------------------------------------
// One round r of the hull of hulls reads (cnt, off, list) and writes the survivor counts into nxt; prev holds the
// counts of round r - 1 (nullptr in round 0), so a set that stopped shrinking is carried over unreduced.
__global__ void k_sizes(Params q, int* cnt0) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= q.n_sets; s += gridDim.x * blockDim.x) {
    const int z = s < q.n_sets ? max(q.set_size[(size_t)s * q.size_stride], 0) : 0;
    q.size[s] = z;
    cnt0[s] = z;
  }
}

// after the scan of size into start: a set reaching past n is ST_BAD and takes no points; round-0 list = identity
__global__ void k_init(Params q, int* cnt0) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, str = (long long)gridDim.x * blockDim.x;
  for (long long s = tid; s < q.n_sets; s += str) {
    const bool bad = (long long)q.start[s] + q.size[s] > q.n;
    q.status[s] = bad ? ST_BAD : (q.size[s] < 4 ? ST_TOO_FEW : ST_OK);
    if (bad) cnt0[s] = 0;
    q.vertex_count[s] = 0;
    q.facet_count[s] = 0;
  }
  for (long long i = tid; i < q.n; i += str) {
    q.list[0][i] = (int)i;
    q.is_vertex[i] = 0;
    q.mark[i] = 0;
  }
}

__global__ void k_tiles(Params q, const int* cnt, const int* prev, int* red, int* nxt) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= q.n_sets; s += gridDim.x * blockDim.x) {
    nxt[s] = 0;
    if (s == q.n_sets) { q.ntile[s] = 0; continue; }
    const int c = cnt[s];
    red[s] = q.status[s] == ST_OK && c > TILE && (prev == nullptr || c < prev[s]);
    q.ntile[s] = red[s] ? (c + TILE - 1) / TILE : 1;
  }
}

__global__ void __launch_bounds__(NT) k_tile(Params q, const int* cnt, const int* off, const int* list, const int* red,
                                             int* nxt) {
  __shared__ Smem sm;
  __shared__ int kept;
  const int t = blockIdx.x;
  if (t >= q.tile_start[q.n_sets]) return;
  int lo = 0, hi = q.n_sets - 1;                             // last set with tile_start <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (q.tile_start[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const int s = lo, c = cnt[s], j = t - q.tile_start[s];
  const bool rd = red[s] != 0;
  const int b = rd ? j * TILE : 0, m = rd ? min(TILE, c - b) : c;
  const int* ids = list + off[s] + b;
  if (threadIdx.x == 0) kept = 0;
  for (int i = threadIdx.x; i < m; i += NT) q.mark[ids[i]] = rd ? 0 : 1;
  __syncthreads();
  int st = ST_FLAT;
  if (rd) {
    const Work w = work_at(q, 2 * (long long)(off[s] + b) + 8 * (long long)t);
    st = hull_list(q.pts, ids, m, w, sm, q.start_at, q.end_at, [&](int v) { q.mark[v] = 1; atomicAdd(&kept, 1); });
    if (st != ST_OK)
      for (int i = threadIdx.x; i < m; i += NT) q.mark[ids[i]] = 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) atomicAdd(&nxt[s], st == ST_OK ? kept : m);
}

__global__ void k_keep(Params q, const int* off, const int* list) {
  const long long total = min((long long)off[q.n_sets], q.n);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += (long long)gridDim.x * blockDim.x)
    q.keep[i] = i < total ? q.mark[list[i]] : 0;
}

__global__ void __launch_bounds__(NT) k_final(Params q, const int* cnt, const int* off, const int* list) {
  __shared__ Smem sm;
  const int s = blockIdx.x;
  if (q.status[s] != ST_OK) return;
  const int c = cnt[s], o = off[s];
  const int* ids = list + o;
  const Work w = work_at(q, 2 * (long long)o + 8 * (long long)s);
  if (threadIdx.x == 0) sm.nvert = 0;
  __syncthreads();
  const int st = hull_list(q.pts, ids, c, w, sm, q.start_at, q.end_at,
                           [&](int v) { q.is_vertex[v] = 1; atomicAdd(&sm.nvert, 1); });
  if (st != ST_OK) {
    if (threadIdx.x == 0) q.status[s] = st;
    return;
  }
  const int hw = sm.hw;
  if (threadIdx.x == 0) {                                    // slot -> output row, in slot order
    int k = 0;
    for (int f = 0; f < hw; ++f) w.vis[f] = w.fs[f] == ALIVE ? k++ : -1;
    sm.nf = k;
    q.vertex_count[s] = sm.nvert;
    q.facet_count[s] = k;
  }
  __syncthreads();
  const long long row0 = 2 * (long long)q.start[s];
  for (int f = threadIdx.x; f < hw; f += NT) {
    const int k = w.vis[f];
    if (k < 0) continue;
    for (int j = 0; j < 3; ++j) {
      q.facets[3 * (row0 + k) + j] = w.fv[3 * f + j];
      if (q.facet_nbr) q.facet_nbr[3 * (row0 + k) + j] = w.vis[w.fn[3 * f + j]];
    }
  }
}

// ---- minimum-volume box ---------------------------------------------------------------------------------------------
struct ObbParams {
  const double* pts;
  const int* facets; const int* facet_nbr; const int* facet_count;
  const int* vertices; const int* vertex_count; const int* status;
  double* box; int* box_status;
  double* nr; double* nu;   // [cap][3] rounded and unit normals
  double* res;              // [cap][9] vol, d0, d1, lo0, lo1, hi0, hi1, hmin, hmax
};

__device__ __forceinline__ double3 sub3(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double3 cross3(double3 a, double3 b) {
  return make_double3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ double dot3(double3 a, double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ double round10(double x) { return rint(x * 1e10) / 1e10; }

__device__ __forceinline__ void basis(double3 n, double3& b1, double3& b2) {
  b1 = cross3(n, fabs(n.x) < 0.9 ? make_double3(1.0, 0.0, 0.0) : make_double3(0.0, 1.0, 0.0));
  const double l = sqrt(dot3(b1, b1));
  b1 = make_double3(b1.x / l, b1.y / l, b1.z / l);
  b2 = cross3(n, b1);
}

__global__ void k_obb_normals(ObbParams q) {
  if (*q.status != ST_OK) return;
  const int F = *q.facet_count;
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < F; f += gridDim.x * blockDim.x) {
    const double3 a = ld(q.pts, q.facets[3 * f]), b = ld(q.pts, q.facets[3 * f + 1]), c = ld(q.pts, q.facets[3 * f + 2]);
    const double3 N = cross3(sub3(b, a), sub3(c, a));
    const double l = sqrt(dot3(N, N));
    const double3 u = make_double3(N.x / l, N.y / l, N.z / l);
    q.nu[3 * f] = u.x; q.nu[3 * f + 1] = u.y; q.nu[3 * f + 2] = u.z;
    q.nr[3 * f] = round10(u.x); q.nr[3 * f + 1] = round10(u.y); q.nr[3 * f + 2] = round10(u.z);
  }
}

__global__ void __launch_bounds__(NT) k_obb_eval(ObbParams q) {
  if (*q.status != ST_OK) return;
  const int F = *q.facet_count, V = *q.vertex_count;
  __shared__ int dup;
  __shared__ double rd[NT][8];
  for (int f = blockIdx.x; f < F; f += gridDim.x) {
    const double3 n = make_double3(q.nr[3 * f], q.nr[3 * f + 1], q.nr[3 * f + 2]);
    if (threadIdx.x == 0) dup = 0;
    __syncthreads();
    for (int g = threadIdx.x; g < f; g += NT)
      if (q.nr[3 * g] == n.x && q.nr[3 * g + 1] == n.y && q.nr[3 * g + 2] == n.z) dup = 1;
    __syncthreads();
    if (dup) {
      if (threadIdx.x == 0) q.res[9 * (size_t)f] = INFINITY;
      __syncthreads();
      continue;
    }
    double3 b1, b2;
    basis(n, b1, b2);
    double hmin = INFINITY, hmax = -INFINITY;
    for (int i = threadIdx.x; i < V; i += NT) {
      const double h = dot3(ld(q.pts, q.vertices[i]), n);
      hmin = fmin(hmin, h);
      hmax = fmax(hmax, h);
    }
    // best rectangle over this thread's silhouette edges: area, edge id, d0, d1, lo0, lo1, hi0, hi1
    double best[8] = {INFINITY, 0, 0, 0, 0, 0, 0, 0};
    for (int e = threadIdx.x; e < 3 * F; e += NT) {
      const int g = e / 3, j = e % 3, o = q.facet_nbr[3 * g + j];
      if (o < g) continue;
      const double sg = q.nu[3 * g] * n.x + q.nu[3 * g + 1] * n.y + q.nu[3 * g + 2] * n.z;
      const double so = q.nu[3 * o] * n.x + q.nu[3 * o + 1] * n.y + q.nu[3 * o + 2] * n.z;
      const double tol = 1e-9;
      if (!((sg >= -tol && so <= tol) || (sg <= tol && so >= -tol))) continue;
      const double3 pa = ld(q.pts, q.facets[3 * g + j]), pb = ld(q.pts, q.facets[3 * g + (j + 1) % 3]);
      const double ex = dot3(pb, b1) - dot3(pa, b1), ey = dot3(pb, b2) - dot3(pa, b2);
      const double ln = sqrt(ex * ex + ey * ey);
      if (!(ln > 0.0)) continue;
      const double d0 = ex / ln, d1 = ey / ln;
      double ulo = INFINITY, uhi = -INFINITY, wlo = INFINITY, whi = -INFINITY;
      for (int i = 0; i < V; ++i) {
        const double3 p = ld(q.pts, q.vertices[i]);
        const double x = dot3(p, b1), y = dot3(p, b2);
        const double u = x * d0 + y * d1, w = x * -d1 + y * d0;
        ulo = fmin(ulo, u); uhi = fmax(uhi, u); wlo = fmin(wlo, w); whi = fmax(whi, w);
      }
      const double area = (uhi - ulo) * (whi - wlo);
      if (area < best[0]) {
        best[0] = area; best[1] = e; best[2] = d0; best[3] = d1;
        best[4] = ulo; best[5] = wlo; best[6] = uhi; best[7] = whi;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      hmin = fmin(hmin, __shfl_xor_sync(0xffffffffu, hmin, o));
      hmax = fmax(hmax, __shfl_xor_sync(0xffffffffu, hmax, o));
    }
    for (int k = 0; k < 8; ++k) rd[threadIdx.x][k] = best[k];
    __shared__ double wh[NT / 32][2];
    if ((threadIdx.x & 31) == 0) { wh[threadIdx.x >> 5][0] = hmin; wh[threadIdx.x >> 5][1] = hmax; }
    __syncthreads();
    if (threadIdx.x == 0) {
      int bi = 0;
      for (int t = 1; t < NT; ++t)
        if (rd[t][0] < rd[bi][0] || (rd[t][0] == rd[bi][0] && rd[t][1] < rd[bi][1])) bi = t;
      for (int k = 1; k < NT / 32; ++k) { hmin = fmin(hmin, wh[k][0]); hmax = fmax(hmax, wh[k][1]); }
      double* r = q.res + 9 * (size_t)f;
      r[0] = rd[bi][0] * (hmax - hmin);
      for (int k = 0; k < 6; ++k) r[1 + k] = rd[bi][2 + k];
      r[7] = hmin; r[8] = hmax;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ bool lex_less(const double* a, const double* b) {
  for (int k = 0; k < 3; ++k) {
    if (a[k] < b[k]) return true;
    if (a[k] > b[k]) return false;
  }
  return false;
}

__global__ void __launch_bounds__(NT) k_obb_pick(ObbParams q) {
  const int st = *q.status;
  const int F = st == ST_OK ? *q.facet_count : 0;
  __shared__ int cand[NT];
  int bi = -1;
  for (int f = threadIdx.x; f < F; f += NT) {
    const double v = q.res[9 * (size_t)f];
    if (!(v < INFINITY)) continue;
    if (bi < 0 || v < q.res[9 * (size_t)bi] || (v == q.res[9 * (size_t)bi] && lex_less(q.nr + 3 * f, q.nr + 3 * bi))) bi = f;
  }
  cand[threadIdx.x] = bi;
  __syncthreads();
  if (threadIdx.x != 0) return;
  bi = -1;
  for (int t = 0; t < NT; ++t) {
    const int f = cand[t];
    if (f < 0) continue;
    if (bi < 0 || q.res[9 * (size_t)f] < q.res[9 * (size_t)bi] ||
        (q.res[9 * (size_t)f] == q.res[9 * (size_t)bi] && lex_less(q.nr + 3 * f, q.nr + 3 * bi)))
      bi = f;
  }
  if (bi < 0) {
    *q.box_status = st == ST_OK ? ST_FLAT : st;
    return;
  }
  const double* r = q.res + 9 * (size_t)bi;
  double3 n = make_double3(q.nr[3 * bi], q.nr[3 * bi + 1], q.nr[3 * bi + 2]), b1, b2;
  basis(n, b1, b2);
  const double d0 = r[1], d1 = r[2];
  const double3 a0 = make_double3(d0 * b1.x + d1 * b2.x, d0 * b1.y + d1 * b2.y, d0 * b1.z + d1 * b2.z);
  const double3 a1 = make_double3(-d1 * b1.x + d0 * b2.x, -d1 * b1.y + d0 * b2.y, -d1 * b1.z + d0 * b2.z);
  double mid[3] = {(r[3] + r[5]) / 2, (r[4] + r[6]) / 2, (r[8] + r[7]) / 2};
  const double ext[3] = {r[5] - r[3], r[6] - r[4], r[8] - r[7]};
  if (dot3(cross3(a0, a1), n) < 0.0) {
    n = make_double3(-n.x, -n.y, -n.z);
    mid[2] = -mid[2];
  }
  const double R[3][3] = {{a0.x, a1.x, n.x}, {a0.y, a1.y, n.y}, {a0.z, a1.z, n.z}};
  for (int i = 0; i < 3; ++i) {
    q.box[i] = R[i][0] * mid[0] + R[i][1] * mid[1] + R[i][2] * mid[2];
    for (int j = 0; j < 3; ++j) q.box[3 + 3 * i + j] = R[i][j];
    q.box[12 + i] = ext[i];
  }
  *q.box_status = ST_OK;
}

// ---- handle scratch (DeviceBuffer's rule) -------------------------------------------------------------------------
struct Workspace {
  DeviceBuffer<unsigned char> buf;
  DeviceBuffer<void> cub_tmp;
  DeviceBuffer<double> obb;
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace hull
