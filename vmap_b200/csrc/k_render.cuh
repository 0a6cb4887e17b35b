// View rendering of the object map (K9): ray / box culling, per-box sample emission and front-to-back compositing
// of many object networks into one camera view (vmap_b200/render.py, oracle/render_oracle.py mirrors it).
//
// The rule (the reference has no compositional renderer; every convention is one the package already has):
//   Sources.  Source s is one object network with an oriented box: centre c, axes R (columns, R stored row-major),
//     half-extents h = extent / (2 * bound_extent) (Trainer.meshing's box), a point offset `off` (obj_center) and an
//     obj_id.  Table row: c[3], R[9], h[3], off[3] as fp64.
//   Rays.  Pixel (u, v) of a W x H camera is ray r = u*H + v (images are [W, H]).  All geometry is fp64 with every
//     operation rounded on its own (no FMA contraction), in exactly this order:
//       dcx = (u - cx) / fx;  dcy = (v - cy) / fy
//       d_j = (T[j][0]*dcx + T[j][1]*dcy) + T[j][2];   o_j = T[j][3]          (T = T_wc rows 0..2)
//     The ray parameter t is camera z-depth (the training depth convention).
//   Hits.  q_j = o_j - c_j;  o'_i = (R[0][i]*q_0 + R[1][i]*q_1) + R[2][i]*q_2;  d'_i likewise with d.
//     Per axis i: d'_i == 0 -> inside the slab iff |o'_i| <= h_i (else no hit);
//                 otherwise a = (-h_i - o'_i) / d'_i, b = (h_i - o'_i) / d'_i, lo = min(a, b), hi = max(a, b).
//     t0 = max(near, lo_0, lo_1, lo_2) + 0.0, t1 = min(far, hi_0, hi_1, hi_2) + 0.0 (the + 0.0 turns -0.0 into +0.0);
//     a hit iff t0 < t1.  A ray keeps the nearest
//     VMB_RENDER_MAX_HITS hits by (t0, source index), sorted that way; rays with more count as overflow.
//   Coarse samples.  w = (t1 - t0) / n_coarse; z_k = t0 + (k + 0.5) * w; p_j = o_j + z_k * d_j (fp64), then
//     point = float(p_j) - float(off_j) and z = float(z_k).
//   Fine samples (rays with a surface z*, fp32 from the coarse composite).  zs = double(z*),
//     y_k = (zs - eps) + (k + 0.5) * ((eps + eps) / n_fine); hit (t0, t1) evaluates every y_k with t0 <= y_k <= t1.
//   Compositing (fp32).  All samples of a ray merge into one sequence ascending in z, ties by source index, then pass
//     (coarse first), then k.  occ = sigmoid(alpha); T_i = occ_i * prod_{j<i}(1 - occ_j + 1e-10);
//     depth = sum T z, colour = sum T c, opacity = sum T (render_rays.py:26-51).  The surface sample is the first
//     whose running opacity reaches 0.5: z* = its z, instance = its source's obj_id; otherwise -1 and no z*
//     (z* is stored as -1: every real sample has z > t0 >= near >= 0).
//   Layout.  A pass's samples are source-major: source, then ascending ray, then k.  A (ray, hit) entry's first
//     sample is base[ray][hit]; entries are ordered by a stable radix sort on the source index, so the order is
//     fixed.  No floating-point atomics: output is bitwise reproducible and independent of the ray chunking.
#pragma once
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#define VMB_RENDER_MAX_HITS 16
#define VMB_RENDER_MAX_SRC 1024
#define VMB_RENDER_BOX 18

namespace render {

struct Params {
  int W, H;
  double fx, fy, cx, cy, T[12];
  double near_, far_, eps;
  int n_src;
  const double* boxes;        // device [n_src][18] (workspace copy)
  const int* obj_id;          // device [n_src]
  long long ray0;
  int n_rays, n_coarse, n_fine, pass;
  int* hit_src; double* hit_t; int* hit_count; int* overflow; int* src_total;
  float* zstar; int* surf;
  // emit / sort scratch
  int* keys; int* keys_alt; int* vals; int* vals_alt; int* cnt; int* wbase;
  float* points; float* z; int* base;
  const float *z_c, *alpha_c, *colour_c; const int* base_c;
  const float *z_f, *alpha_f, *colour_f; const int* base_f;
  float *depth, *colour, *opacity; int* instance;
};

__device__ __forceinline__ void ray_of(const Params& q, int r, double o[3], double d[3]) {
  const long long g = q.ray0 + r;
  const double u = (double)(g / q.H), v = (double)(g % q.H);
  const double dcx = __ddiv_rn(__dsub_rn(u, q.cx), q.fx), dcy = __ddiv_rn(__dsub_rn(v, q.cy), q.fy);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    d[j] = __dadd_rn(__dadd_rn(__dmul_rn(q.T[4 * j], dcx), __dmul_rn(q.T[4 * j + 1], dcy)), q.T[4 * j + 2]);
    o[j] = q.T[4 * j + 3];
  }
}

__device__ __forceinline__ bool slab(const double* b, const double o[3], const double d[3], double near_, double far_,
                                     double& t0, double& t1) {
  const double q0 = __dsub_rn(o[0], b[0]), q1 = __dsub_rn(o[1], b[1]), q2 = __dsub_rn(o[2], b[2]);
  t0 = near_; t1 = far_;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double op = __dadd_rn(__dadd_rn(__dmul_rn(b[3 + i], q0), __dmul_rn(b[6 + i], q1)), __dmul_rn(b[9 + i], q2));
    const double dp = __dadd_rn(__dadd_rn(__dmul_rn(b[3 + i], d[0]), __dmul_rn(b[6 + i], d[1])), __dmul_rn(b[9 + i], d[2]));
    const double h = b[12 + i];
    if (dp == 0.0) {
      if (!(fabs(op) <= h)) return false;
    } else {
      const double a = __ddiv_rn(__dsub_rn(-h, op), dp), c = __ddiv_rn(__dsub_rn(h, op), dp);
      t0 = fmax(t0, fmin(a, c));
      t1 = fmin(t1, fmax(a, c));
    }
  }
  t0 = __dadd_rn(t0, 0.0);                 // -0.0 -> +0.0: the sign of a zero bound does not depend on fmax's choice
  t1 = __dadd_rn(t1, 0.0);
  return t0 < t1;
}

// pass 0: one thread per ray; the nearest MAX_HITS hits by (t0, source), sorted
__global__ void __launch_bounds__(128) k_cull(Params q) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= q.n_rays) return;
  double o[3], d[3];
  ray_of(q, r, o, d);
  int hs[VMB_RENDER_MAX_HITS];
  double h0[VMB_RENDER_MAX_HITS], h1[VMB_RENDER_MAX_HITS];
  int n = 0, total = 0;
  for (int s = 0; s < q.n_src; ++s) {
    double t0, t1;
    if (!slab(q.boxes + (size_t)s * VMB_RENDER_BOX, o, d, q.near_, q.far_, t0, t1)) continue;
    ++total;
    if (n == VMB_RENDER_MAX_HITS && !(t0 < h0[n - 1])) continue;       // ties lose: s is the largest index so far
    int i = (n < VMB_RENDER_MAX_HITS) ? n++ : n - 1;
    while (i > 0 && t0 < h0[i - 1]) { hs[i] = hs[i - 1]; h0[i] = h0[i - 1]; h1[i] = h1[i - 1]; --i; }
    hs[i] = s; h0[i] = t0; h1[i] = t1;
  }
  const size_t e = (size_t)r * VMB_RENDER_MAX_HITS;
  for (int i = 0; i < VMB_RENDER_MAX_HITS; ++i) {
    q.hit_src[e + i] = i < n ? hs[i] : -1;
    q.hit_t[2 * (e + i)] = i < n ? h0[i] : 0.0;
    q.hit_t[2 * (e + i) + 1] = i < n ? h1[i] : 0.0;
  }
  q.hit_count[r] = n;
  if (total > VMB_RENDER_MAX_HITS) atomicAdd(q.overflow, 1);
}

// fine positions of one hit: the k range [k0, k1) with t0 <= y_k <= t1 (y_k is non-decreasing in k)
__device__ __forceinline__ double fine_pos(double zs, double eps, int n_fine, int k) {
  return __dadd_rn(__dsub_rn(zs, eps), __dmul_rn((double)k + 0.5, __ddiv_rn(__dadd_rn(eps, eps), (double)n_fine)));
}
__device__ __forceinline__ int fine_range(const Params& q, float zstar, double t0, double t1, int& k0) {
  k0 = 0;
  if (!(zstar >= 0.f)) return 0;
  const double zs = (double)zstar;
  int n = 0;
  for (int k = 0; k < q.n_fine; ++k) {
    const double y = fine_pos(zs, q.eps, q.n_fine, k);
    if (t0 <= y && y <= t1) { if (n == 0) k0 = k; ++n; }
  }
  return n;
}

__device__ __forceinline__ int entry_count(const Params& q, int r, int i, int& k0) {
  const size_t e = (size_t)r * VMB_RENDER_MAX_HITS + i;
  k0 = 0;
  if (i >= q.hit_count[r]) return 0;
  if (q.pass == 0) return q.n_coarse;
  return fine_range(q, q.zstar[r], q.hit_t[2 * e], q.hit_t[2 * e + 1], k0);
}

// one thread per (ray, hit) entry: sort key (source, or n_src for an empty slot), sample count, per-source totals
__global__ void k_entry_counts(Params q) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n_e = (long long)q.n_rays * VMB_RENDER_MAX_HITS;
  if (e > n_e) return;
  if (e == n_e) { q.cnt[e] = 0; return; }
  const int r = (int)(e / VMB_RENDER_MAX_HITS), i = (int)(e % VMB_RENDER_MAX_HITS);
  int k0;
  const int c = entry_count(q, r, i, k0);
  const int s = i < q.hit_count[r] ? q.hit_src[e] : q.n_src;
  q.keys[e] = (c > 0) ? s : q.n_src;
  q.vals[e] = (int)e;
  q.cnt[e] = c;
  if (c > 0) atomicAdd(q.src_total + s, c);
}

// counts in source-major order, ready for the exclusive scan
__global__ void k_gather_counts(Params q, const int* sorted_vals, const int* cnt, int* out) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n_e = (long long)q.n_rays * VMB_RENDER_MAX_HITS;
  if (j > n_e) return;
  out[j] = (j == n_e) ? 0 : cnt[sorted_vals[j]];
}
__global__ void k_scatter_base(Params q, const int* sorted_vals, const int* scanned, int* wbase) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)q.n_rays * VMB_RENDER_MAX_HITS) return;
  wbase[sorted_vals[j]] = scanned[j];
}

// one thread per (ray, hit) entry: base index, points and z of its samples
__global__ void k_emit(Params q) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)q.n_rays * VMB_RENDER_MAX_HITS) return;
  const int r = (int)(e / VMB_RENDER_MAX_HITS), i = (int)(e % VMB_RENDER_MAX_HITS);
  int k0;
  const int c = entry_count(q, r, i, k0);
  const int b = q.wbase[e];
  q.base[e] = b;
  if (c == 0) return;
  double o[3], d[3];
  ray_of(q, r, o, d);
  const double* bx = q.boxes + (size_t)q.hit_src[e] * VMB_RENDER_BOX;
  const float off0 = (float)bx[15], off1 = (float)bx[16], off2 = (float)bx[17];
  const double t0 = q.hit_t[2 * e], t1 = q.hit_t[2 * e + 1];
  const double w = __ddiv_rn(__dsub_rn(t1, t0), (double)q.n_coarse);
  const double zs = (double)q.zstar[r];
  for (int j = 0; j < c; ++j) {
    const double zk = (q.pass == 0) ? __dadd_rn(t0, __dmul_rn((double)j + 0.5, w)) : fine_pos(zs, q.eps, q.n_fine, k0 + j);
    const size_t p = (size_t)b + j;
    q.points[3 * p] = (float)__dadd_rn(o[0], __dmul_rn(zk, d[0])) - off0;
    q.points[3 * p + 1] = (float)__dadd_rn(o[1], __dmul_rn(zk, d[1])) - off1;
    q.points[3 * p + 2] = (float)__dadd_rn(o[2], __dmul_rn(zk, d[2])) - off2;
    q.z[p] = (float)zk;
  }
}

// one thread per ray: merge the ray's sample lists ((z, source, pass) order) and composite front to back
__global__ void __launch_bounds__(128) k_composite(Params q) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= q.n_rays) return;
  const int nh = q.hit_count[r];
  const bool fine = q.pass == 1;
  const float zst = fine ? q.zstar[r] : -1.f;
  int pos[2 * VMB_RENDER_MAX_HITS], end[2 * VMB_RENDER_MAX_HITS];
  const size_t e0 = (size_t)r * VMB_RENDER_MAX_HITS;
  for (int i = 0; i < nh; ++i) {
    pos[i] = q.base_c[e0 + i];
    end[i] = pos[i] + q.n_coarse;
    int k0 = 0, c = 0;
    if (fine) c = fine_range(q, zst, q.hit_t[2 * (e0 + i)], q.hit_t[2 * (e0 + i) + 1], k0);
    pos[VMB_RENDER_MAX_HITS + i] = fine ? q.base_f[e0 + i] : 0;
    end[VMB_RENDER_MAX_HITS + i] = pos[VMB_RENDER_MAX_HITS + i] + c;
  }
  float hz[2 * VMB_RENDER_MAX_HITS];         // z of each list's head (+inf when the list is done)
  for (int l = 0; l < 2 * VMB_RENDER_MAX_HITS; ++l) {
    const int i = l % VMB_RENDER_MAX_HITS;
    const bool live = i < nh && (l < VMB_RENDER_MAX_HITS || fine) && pos[l] < end[l];
    hz[l] = live ? (l < VMB_RENDER_MAX_HITS ? q.z_c : q.z_f)[pos[l]] : INFINITY;
  }
  int hsrc[VMB_RENDER_MAX_HITS];
  for (int i = 0; i < nh; ++i) hsrc[i] = q.hit_src[e0 + i];
  float prod = 1.f, acc_d = 0.f, acc_o = 0.f, acc_c0 = 0.f, acc_c1 = 0.f, acc_c2 = 0.f, zsurf = -1.f;
  int n_seen = 0, surf = -1, inst = -1;
  for (;;) {
    int best = -1;
    float bz = 0.f;
    int bs = 0;
    const int n_lists = fine ? 2 * nh : nh;
    for (int j = 0; j < n_lists; ++j) {
      const int l = j < nh ? j : VMB_RENDER_MAX_HITS + (j - nh);
      const float zl = hz[l];
      if (zl == INFINITY) continue;
      const int sl = hsrc[l % VMB_RENDER_MAX_HITS];
      // lists are scanned coarse-first, so (z, source) ties keep the coarse list
      if (best < 0 || zl < bz || (zl == bz && sl < bs)) { best = l; bz = zl; bs = sl; }
    }
    if (best < 0) break;
    const bool is_c = best < VMB_RENDER_MAX_HITS;
    const int p = pos[best]++;
    hz[best] = pos[best] < end[best] ? (is_c ? q.z_c : q.z_f)[pos[best]] : INFINITY;
    const float a = (is_c ? q.alpha_c : q.alpha_f)[p];
    const float* cc = (is_c ? q.colour_c : q.colour_f) + 3 * (size_t)p;
    const float occ = 1.0f / (1.0f + expf(-a));
    const float T = occ * prod;
    prod = prod * ((1.0f - occ) + 1e-10f);
    acc_d += T * bz;
    acc_c0 += T * cc[0]; acc_c1 += T * cc[1]; acc_c2 += T * cc[2];
    acc_o += T;
    if (surf < 0 && acc_o >= 0.5f) { surf = n_seen; zsurf = bz; inst = q.obj_id[bs]; }
    ++n_seen;
  }
  if (!fine) { q.zstar[r] = zsurf; q.surf[r] = surf; }
  if (fine || q.n_fine == 0) {
    const long long g = q.ray0 + r;
    q.depth[g] = acc_d; q.opacity[g] = acc_o; q.instance[g] = inst;
    q.colour[3 * g] = acc_c0; q.colour[3 * g + 1] = acc_c1; q.colour[3 * g + 2] = acc_c2;
  }
}

struct Workspace {
  DeviceBuffer<double> boxes;
  DeviceBuffer<int> obj_id;
  DeviceBuffer<int> ints;                             // keys | keys_alt | vals | vals_alt | cnt | scan | wbase
  DeviceBuffer<void> cub_tmp;
  Params last{};                                      // the last count (emit must match it)
  bool counted = false;
};

inline unsigned blocks_for(long long n, int bs) { return (unsigned)((n + bs - 1) / bs); }

}  // namespace render
