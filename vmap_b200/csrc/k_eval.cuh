// K6: 3-D reconstruction metrics (metric/eval_3D_obj.py, eval_3D_scene.py, metrics.py): box crop of a triangle mesh,
// area-weighted surface sampling and exact nearest-neighbour distances.  Means and ratios over the distances are torch
// reductions in vmap_b200/metrics.py; every kernel here does one job.
//
// Box crop (trimesh.Trimesh.slice_plane with the six faces of a box): one thread per face clips the triangle against
// the box's six half-spaces with Sutherland-Hodgman in fp64 (at most 3 + 6 = 9 vertices) and fan-triangulates the
// result from its first vertex.  Planes in the order (axis 0, +), (axis 0, -), (axis 1, +), ...; along each polygon
// edge (a, b) the clipper emits a when d(a) >= 0 and then the crossing a + t (b - a), t = d(a) / (d(a) - d(b)), when a
// and b lie on different sides.  Count / emit with one host sync between them, as marching cubes: the count pass
// writes each face's triangle count into an (F+1)-entry scan, so the output order is (input face, fan order).
//
// Surface sampling (trimesh.sample.sample_surface): fp64 face areas 0.5 |e1 x e2| and their inclusive prefix (CUB),
// then per point searchsorted(side='left') on u0 * total and the reflected barycentric rule
// (r = (u1, u2); r = |r - 1| when u1 + u2 > 1; p = v0 + (r1 e1 + r2 e2)), in fp64, stored as fp32.
//
// Nearest neighbour: the ref points are counting-sorted into a uniform grid over their bounding box (bounding box by
// an order-preserving-key atomic reduction, grid sizing in a one-thread kernel, so nothing waits for the host; about one
// cell per ref point, at most EVAL_MAX_CELLS cells and 1024 per axis).  One thread per query visits the cells of
// growing Chebyshev radius r around the query's clamped cell and stops when every cell not yet visited lies farther
// than the best distance found: the bound is the Euclidean distance from the query to each of the (up to six) boxes
// grid-box ∩ {beyond the visited block on one side}, so queries far outside the ref box stop as soon as nearby cells
// are exhausted.  The search is exact (ties to the lowest ref index).  Cost per query: O(points in the cells within
// the true nearest distance, plus those cells); a cloud that fills its box gives ~1 point per cell and a few dozen
// cells, a surface sample of n points ~n^(1/3) points per occupied cell.  Worst case (all ref points in one cell,
// e.g. one tight blob plus far outliers that stretch the box): O(n_ref + cells) per query, i.e. brute force.
#pragma once
#include "common.cuh"
#include "k_sampler.cuh"                       // philox4x32_10
#include <cub/device/device_scan.cuh>

namespace eval3d {

constexpr int EVAL_MAX_CELLS = 1 << 22;
constexpr int EVAL_MAX_AXIS = 1024;
constexpr int CLIP_MAX_POLY = 9;

// ---- box crop -------------------------------------------------------------------------------------------------------
struct ClipParams {
  const float* v; long long nv;
  const int* f; long long nf;
  float c[3], ax[3][3], half[3];   // center, box axes (ax[j] = axis j), half extents
  int* scan;                       // [nf+1] triangle counts -> first triangle of each face
  float* out; long long max_tri;   // [T][3][3]
};

__device__ __forceinline__ bool clip_face_ok(const ClipParams& q, long long fi, int (&id)[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    id[k] = __ldg(q.f + 3 * fi + k);
    if (id[k] < 0 || id[k] >= q.nv) return false;
  }
  return true;
}

// Clips face fi in place into P[0..n); returns n (0 when nothing is left or the face has an out-of-range index).
// The polygon is kept in fp64 (fp32 in and out): a crossing d(a) / (d(a) - d(b)) near a plane cancels, and fp64 keeps
// the emitted vertices within rounding of the exact clip.
__device__ __forceinline__ int clip_face(const ClipParams& q, long long fi, double3 (&P)[CLIP_MAX_POLY]) {
  int id[3];
  if (!clip_face_ok(q, fi, id)) return 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float* p = q.v + 3 * (long long)id[k];
    P[k] = make_double3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
  }
  int n = 3;
  double3 Q[CLIP_MAX_POLY];
  for (int pl = 0; pl < 6 && n > 0; ++pl) {
    const int j = pl >> 1;
    const double sg = (pl & 1) ? -1.0 : 1.0;
    const double ax = q.ax[j][0], ay = q.ax[j][1], az = q.ax[j][2];
    const double cx = q.c[0], cy = q.c[1], cz = q.c[2], hj = q.half[j];
    auto dist = [&](double3 p) {
      const double s = __dadd_rn(__dadd_rn(__dmul_rn(p.x - cx, ax), __dmul_rn(p.y - cy, ay)), __dmul_rn(p.z - cz, az));
      return hj - sg * s;
    };
    int m = 0;
    double da = dist(P[0]);
    for (int k = 0; k < n; ++k) {
      const double3 a = P[k], b = P[k + 1 < n ? k + 1 : 0];
      const double db = dist(b);
      if (da >= 0.0 && m < CLIP_MAX_POLY) Q[m++] = a;
      if ((da >= 0.0) != (db >= 0.0) && m < CLIP_MAX_POLY) {
        const double t = da / (da - db);
        Q[m++] = make_double3(a.x + t * (b.x - a.x), a.y + t * (b.y - a.y), a.z + t * (b.z - a.z));
      }
      da = db;
    }
    n = m;
    for (int k = 0; k < n; ++k) P[k] = Q[k];
  }
  return n;
}

__global__ void __launch_bounds__(128) k_clip_count(ClipParams q) {
  const long long fi = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (fi > q.nf) return;
  if (fi == q.nf) { q.scan[fi] = 0; return; }
  double3 P[CLIP_MAX_POLY];
  const int n = clip_face(q, fi, P);
  q.scan[fi] = n >= 3 ? n - 2 : 0;
}

__global__ void __launch_bounds__(128) k_clip_emit(ClipParams q) {
  const long long fi = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (fi >= q.nf) return;
  double3 P[CLIP_MAX_POLY];
  const int n = clip_face(q, fi, P);
  long long t = q.scan[fi];
  for (int k = 1; k + 1 < n; ++k, ++t) {
    if (t >= q.max_tri) break;
    float* o = q.out + 9 * t;
    o[0] = (float)P[0].x; o[1] = (float)P[0].y; o[2] = (float)P[0].z;
    o[3] = (float)P[k].x; o[4] = (float)P[k].y; o[5] = (float)P[k].z;
    o[6] = (float)P[k + 1].x; o[7] = (float)P[k + 1].y; o[8] = (float)P[k + 1].z;
  }
}

// ---- surface sampling -----------------------------------------------------------------------------------------------
struct SampleSurfParams {
  const float* v; long long nv;
  const int* f; long long nf;
  long long n;
  unsigned long long seed;
  const double* uniforms;          // optional [n][3]
  double* cum;                     // [nf] areas -> inclusive prefix
  int* bad;                        // set when a face index is out of range
  float* points; int* face_index;
};

__global__ void __launch_bounds__(256) k_face_area(SampleSurfParams q) {
  const long long fi = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (fi >= q.nf) return;
  int id[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    id[k] = __ldg(q.f + 3 * fi + k);
    if (id[k] < 0 || id[k] >= q.nv) { *q.bad = 1; q.cum[fi] = 0.0; return; }
  }
  double p[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) p[k][r] = (double)__ldg(q.v + 3 * (long long)id[k] + r);
  const double e1x = p[1][0] - p[0][0], e1y = p[1][1] - p[0][1], e1z = p[1][2] - p[0][2];
  const double e2x = p[2][0] - p[0][0], e2y = p[2][1] - p[0][1], e2z = p[2][2] - p[0][2];
  const double cx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
  const double cy = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
  const double cz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
  q.cum[fi] = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz))) * 0.5;
}

__global__ void __launch_bounds__(256) k_sample_surface(SampleSurfParams q) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.n) return;
  double u0, u1, u2;
  if (q.uniforms) {
    u0 = q.uniforms[3 * i]; u1 = q.uniforms[3 * i + 1]; u2 = q.uniforms[3 * i + 2];
  } else {                                   // stream 4 of the project's Philox counters, keyed by the seed
    uint32_t o[4];
    philox4x32_10((uint32_t)i, (uint32_t)(i >> 32), 4u, 0u, (uint32_t)q.seed, (uint32_t)(q.seed >> 32), o);
    u0 = ((double)(o[0] >> 5) * 67108864.0 + (double)(o[1] >> 6)) * (1.0 / 9007199254740992.0);
    u1 = (double)o[2] * (1.0 / 4294967296.0);
    u2 = (double)o[3] * (1.0 / 4294967296.0);
  }
  const double target = __dmul_rn(u0, q.cum[q.nf - 1]);
  long long lo = 0, hi = q.nf;               // first index with cum >= target (numpy searchsorted, side='left')
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (q.cum[mid] < target) lo = mid + 1; else hi = mid;
  }
  const long long fi = lo < q.nf ? lo : q.nf - 1;
  if (u1 + u2 > 1.0) { u1 = fabs(u1 - 1.0); u2 = fabs(u2 - 1.0); }
  const int* fp = q.f + 3 * fi;
  const float* a = q.v + 3 * (long long)__ldg(fp);
  const float* b = q.v + 3 * (long long)__ldg(fp + 1);
  const float* c = q.v + 3 * (long long)__ldg(fp + 2);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double o = (double)__ldg(a + r);
    const double e1 = __dsub_rn((double)__ldg(b + r), o), e2 = __dsub_rn((double)__ldg(c + r), o);
    q.points[3 * i + r] = (float)__dadd_rn(o, __dadd_rn(__dmul_rn(u1, e1), __dmul_rn(u2, e2)));
  }
  if (q.face_index) q.face_index[i] = (int)fi;
}

// ---- nearest neighbour ----------------------------------------------------------------------------------------------
struct Grid {
  double lo[3], h, inv_h;
  int G[3];
};

struct NnParams {
  const float* ref; long long n_ref;
  const float* query; long long n_q;
  unsigned int* keys;              // [6] order-preserving min x,y,z | max x,y,z
  Grid* grid;                      // device
  long long max_cells;
  int* cell_start;                 // [max_cells+1] counts -> exclusive prefix
  int* pt_cell; int* pt_rank;      // [n_ref]
  float4* sorted;                  // [n_ref] x, y, z, original index (bits)
  float* dist; int* index;
};

__device__ __forceinline__ unsigned int fkey(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void __launch_bounds__(256) k_nn_bbox(NnParams q) {
  __shared__ unsigned int s[6];
  if (threadIdx.x < 6) s[threadIdx.x] = threadIdx.x < 3 ? 0xffffffffu : 0u;
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < q.n_ref) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float x = __ldg(q.ref + 3 * i + r);
      if (x == x) { atomicMin(&s[r], fkey(x)); atomicMax(&s[3 + r], fkey(x)); }
    }
  }
  __syncthreads();
  if (threadIdx.x < 3) atomicMin(&q.keys[threadIdx.x], s[threadIdx.x]);
  else if (threadIdx.x < 6) atomicMax(&q.keys[threadIdx.x], s[threadIdx.x]);
}

// One thread: cell edge h for about one ref point per cell of the bounding box (thin axes count as 1/1024 of the
// longest), then grown until the grid fits max_cells.
__global__ void k_nn_grid(NnParams q) {
  Grid g;
  double e[3], emax = 0.0;
  for (int r = 0; r < 3; ++r) {
    const bool any = q.keys[r] != 0xffffffffu;
    g.lo[r] = any ? (double)fkey_inv(q.keys[r]) : 0.0;
    e[r] = any ? (double)fkey_inv(q.keys[3 + r]) - g.lo[r] : 0.0;
    emax = fmax(emax, e[r]);
  }
  if (!(emax > 0.0) || !isfinite(emax)) {
    g.h = 1.0; g.G[0] = g.G[1] = g.G[2] = 1;
  } else {
    double vol = 1.0;
    for (int r = 0; r < 3; ++r) vol *= fmax(e[r], emax / EVAL_MAX_AXIS);
    const double target = (double)min(q.n_ref, q.max_cells);
    double h = fmax(cbrt(vol / target), emax / EVAL_MAX_AXIS);
    for (;;) {
      long long cells = 1;
      for (int r = 0; r < 3; ++r) {
        g.G[r] = max(1, min(EVAL_MAX_AXIS, (int)ceil(e[r] / h)));
        cells *= g.G[r];
      }
      if (cells <= q.max_cells) break;
      h *= 1.0625;
    }
    g.h = h;
  }
  g.inv_h = 1.0 / g.h;
  *q.grid = g;
}

__device__ __forceinline__ int cell_axis(const Grid& g, float x, int r) {
  const double c = floor(((double)x - g.lo[r]) * g.inv_h);
  return c >= (double)g.G[r] ? g.G[r] - 1 : (c > 0.0 ? (int)c : 0);     // NaN -> 0
}

__global__ void __launch_bounds__(256) k_nn_count(NnParams q) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.n_ref) return;
  const Grid g = *q.grid;
  const int cx = cell_axis(g, __ldg(q.ref + 3 * i), 0), cy = cell_axis(g, __ldg(q.ref + 3 * i + 1), 1);
  const int cz = cell_axis(g, __ldg(q.ref + 3 * i + 2), 2);
  const int cell = (cx * g.G[1] + cy) * g.G[2] + cz;
  q.pt_cell[i] = cell;
  q.pt_rank[i] = atomicAdd(q.cell_start + cell, 1);
}

__global__ void __launch_bounds__(256) k_nn_scatter(NnParams q) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.n_ref) return;
  const int pos = q.cell_start[q.pt_cell[i]] + q.pt_rank[i];
  q.sorted[pos] = make_float4(__ldg(q.ref + 3 * i), __ldg(q.ref + 3 * i + 1), __ldg(q.ref + 3 * i + 2),
                              __int_as_float((int)i));
}

__global__ void __launch_bounds__(128) k_nn_query(NnParams q) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.n_q) return;
  const Grid g = *q.grid;
  const float px = __ldg(q.query + 3 * i), py = __ldg(q.query + 3 * i + 1), pz = __ldg(q.query + 3 * i + 2);
  const float p[3] = {px, py, pz};
  const int c[3] = {cell_axis(g, px, 0), cell_axis(g, py, 1), cell_axis(g, pz, 2)};
  // per axis: the query's offset from the grid origin (in cells) and its squared gap to the grid box
  float u[3], gap2[3], base2 = 0.f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    u[a] = (float)(((double)p[a] - g.lo[a]) * g.inv_h);
    const float t = u[a] < 0.f ? -u[a] : (u[a] > (float)g.G[a] ? u[a] - (float)g.G[a] : 0.f);
    gap2[a] = t * t;
    base2 += gap2[a];
  }
  const float h2 = (float)(g.h * g.h);
  float best = __int_as_float(0x7f800000);    // +inf, squared distance
  int best_i = -1;
  const int rmax = max(max(g.G[0], g.G[1]), g.G[2]);
  for (int r = 0; r < rmax; ++r) {
    const int x0 = max(c[0] - r, 0), x1 = min(c[0] + r, g.G[0] - 1);
    const int y0 = max(c[1] - r, 0), y1 = min(c[1] + r, g.G[1] - 1);
    for (int x = x0; x <= x1; ++x) {
      const bool xs = x == c[0] - r || x == c[0] + r;
      for (int y = y0; y <= y1; ++y) {
        const bool face = xs || y == c[1] - r || y == c[1] + r;
        const int zstep = face || r == 0 ? 1 : 2 * r;      // interior (x, y) columns: only z = c -/+ r
        for (int z = c[2] - r; z <= c[2] + r; z += zstep) {
          if (z < 0 || z >= g.G[2]) continue;
          const int cell = (x * g.G[1] + y) * g.G[2] + z;
          const int b = __ldg(q.cell_start + cell), e = __ldg(q.cell_start + cell + 1);
          for (int k = b; k < e; ++k) {
            const float4 s = __ldg(q.sorted + k);
            const float dx = s.x - px, dy = s.y - py, dz = s.z - pz;
            const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            const int id = __float_as_int(s.w);
            if (d2 < best || (d2 == best && id < best_i)) { best = d2; best_i = id; }
          }
        }
      }
    }
    // Lower bound on the distance to every cell outside the visited block [c - r, c + r]: the distance to the part
    // of the grid box beyond the block on one side differs from the distance to the grid box only along that side's
    // axis.  In cell units; shrunk by 1e-4 cell so rounding of the cell assignment can never make it too large.
    float lb2 = __int_as_float(0x7f800000);
    bool more = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (c[a] + r + 1 < g.G[a]) {
        const float t = fmaxf((float)(c[a] + r + 1) - u[a] - 1e-4f, 0.f);
        lb2 = fminf(lb2, base2 - gap2[a] + t * t);
        more = true;
      }
      if (c[a] - r - 1 >= 0) {
        const float t = fmaxf(u[a] - (float)(c[a] - r) - 1e-4f, 0.f);
        lb2 = fminf(lb2, base2 - gap2[a] + t * t);
        more = true;
      }
    }
    if (!more || lb2 * h2 > best) break;
  }
  q.dist[i] = __fsqrt_rn(best);
  if (q.index) q.index[i] = best_i;
}

// Handle-owned, grow-only scratch of the evaluation kernels; the crop scan is kept apart from the rest so sampling or a
// nearest-neighbour query between a crop count and its emit does not disturb the counts.
struct Workspace {
  DeviceBuffer<int> clip_scan;
  DeviceBuffer<double> cum;                              // surface sampling: areas / prefix, then a flag int
  DeviceBuffer<unsigned char> nn;                        // keys | grid | cell_start | pt_cell | pt_rank | sorted
  DeviceBuffer<void> cub_tmp;
  ClipParams last{};                                     // the last crop count (emit must match it)
  bool counted = false;

  cudaError_t exclusive_sum(int* d, long long n, bool capturing, cudaStream_t st) {
    size_t need = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, need, d, (int)n, st);
    if (e == cudaSuccess) e = cub_tmp.grow(need, capturing);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(cub_tmp, need, d, (int)n, st);
    return e;
  }
  cudaError_t inclusive_sum(double* d, long long n, bool capturing, cudaStream_t st) {
    size_t need = 0;
    cudaError_t e = cub::DeviceScan::InclusiveSum(nullptr, need, d, d, (int)n, st);
    if (e == cudaSuccess) e = cub_tmp.grow(need, capturing);
    if (e == cudaSuccess) e = cub::DeviceScan::InclusiveSum(cub_tmp, need, d, d, (int)n, st);
    return e;
  }
};

inline unsigned blocks_for(long long n, int bs) { return (unsigned)((n + bs - 1) / bs); }

}  // namespace eval3d
