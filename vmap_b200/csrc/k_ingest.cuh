// K4: frame ingest -- one GPU pass over the instance image of a new frame.
// Replaces, per frame, the CPU/numpy loop of dataset.py:101-126 (np.unique, one boolean mask per
// instance, get_bbox2d_batch (utils.py:75-84), enlarge_bbox (utils.py:36-57), the
// "inst[obj_ == 0] = 0" relabel) and the per-object state-mask build + full-frame copies of
// train.py:108-141: the frame is written ONCE into a slot of the shared keyframe store and the
// per-object pixel state is derived from the instance id when the sampler reads it.
//
// HBM-bound byte/integer work: algorithmic traffic = 4 B (instance id) [+ 4 B class] per pixel read in
// pass 1, and 4+3+4 B read + 4+4+4 B written per pixel in the store write.  Integer results are exact.
#pragma once
#include "common.cuh"
#include <limits.h>

namespace ing {

constexpr int ST = 8;          // ints per id in the stats table
enum { S_CNT = 0, S_UMIN = 1, S_UMAX1 = 2, S_VMIN = 3, S_VMAX1 = 4, S_CMIN = 5, S_CMAX = 6, S_KEEP = 7 };
constexpr int NSLOT = 128;     // block-local table (ids met by one CTA); overflow goes straight to global atomics

__global__ void k_ingest_init(int* stats, int max_id) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_id) return;
  int* s = stats + (size_t)i * ST;
  s[S_CNT] = 0; s[S_UMIN] = INT_MAX; s[S_UMAX1] = 0; s[S_VMIN] = INT_MAX; s[S_VMAX1] = 0;
  s[S_CMIN] = INT_MAX; s[S_CMAX] = INT_MIN; s[S_KEEP] = 0;
}

__device__ __forceinline__ void flush_global(int* stats, int id, int cnt, int umin, int umax, int vmin, int vmax,
                                             int cmin, int cmax) {
  int* s = stats + (size_t)id * ST;
  atomicAdd(s + S_CNT, cnt);
  atomicMin(s + S_UMIN, umin); atomicMax(s + S_UMAX1, umax + 1);
  atomicMin(s + S_VMIN, vmin); atomicMax(s + S_VMAX1, vmax + 1);
  if (cmin <= cmax) { atomicMin(s + S_CMIN, cmin); atomicMax(s + S_CMAX, cmax); }
}

// pass 1: per-instance pixel count, extent along u (dim 0, image width) and v (dim 1), class range
__global__ void __launch_bounds__(256) k_ingest_stats(const int* __restrict__ inst, const int* __restrict__ cls,
                                                      int W, int Hh, int max_id, int* stats) {
  __shared__ int t_id[NSLOT];
  __shared__ int t_val[NSLOT][7];     // cnt, umin, umax, vmin, vmax, cmin, cmax
  for (int i = threadIdx.x; i < NSLOT; i += blockDim.x) {
    t_id[i] = -2;
    t_val[i][0] = 0; t_val[i][1] = INT_MAX; t_val[i][2] = -1; t_val[i][3] = INT_MAX; t_val[i][4] = -1;
    t_val[i][5] = INT_MAX; t_val[i][6] = INT_MIN;
  }
  __syncthreads();
  const long long n = (long long)W * Hh;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n_round = (n + 31) / 32 * 32;        // whole warps stay converged for the match/reduce ops
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n_round; p += stride) {
    int id = -1, u = 0, v = 0, c = 0;
    if (p < n) { id = inst[p]; u = (int)(p / Hh); v = (int)(p - (long long)u * Hh); if (cls) c = cls[p]; }
    const bool valid = id >= 0 && id < max_id;
    const unsigned grp = __match_any_sync(0xffffffffu, valid ? id : -1);
    const int cnt = __popc(grp);
    const int umin = __reduce_min_sync(grp, u), umax = __reduce_max_sync(grp, u);
    const int vmin = __reduce_min_sync(grp, v), vmax = __reduce_max_sync(grp, v);
    int cmin = INT_MAX, cmax = INT_MIN;
    if (cls) { cmin = __reduce_min_sync(grp, c); cmax = __reduce_max_sync(grp, c); }
    if (!valid || (int)(threadIdx.x & 31) != __ffs(grp) - 1) continue;      // one leader per id per warp
    unsigned h = ((unsigned)id * 2654435761u) >> 25;                          // 7 bits
    int slot = -1;
    for (int probe = 0; probe < NSLOT; ++probe, h = (h + 1) & (NSLOT - 1)) {
      const int old = atomicCAS(&t_id[h], -2, id);
      if (old == -2 || old == id) { slot = (int)h; break; }
    }
    if (slot < 0) { flush_global(stats, id, cnt, umin, umax, vmin, vmax, cmin, cmax); continue; }
    atomicAdd(&t_val[slot][0], cnt);
    atomicMin(&t_val[slot][1], umin); atomicMax(&t_val[slot][2], umax);
    atomicMin(&t_val[slot][3], vmin); atomicMax(&t_val[slot][4], vmax);
    if (cls) { atomicMin(&t_val[slot][5], cmin); atomicMax(&t_val[slot][6], cmax); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NSLOT; i += blockDim.x)
    if (t_id[i] >= 0 && t_val[i][0] > 0)
      flush_global(stats, t_id[i], t_val[i][0], t_val[i][1], t_val[i][2], t_val[i][3], t_val[i][4], t_val[i][5],
                   t_val[i][6]);
}

// per id: drop background-class / too-small instances (dataset.py:106,119), enlarge + clip the box
// (utils.py:36-57), emit it in sceneObject's order [u_lo, u_hi, v_lo, v_hi] (dataset.py:126).
// Instance 0 is the background model: always present with the full image (dataset.py:131).
__global__ void k_ingest_finalize(int* stats, float* bbox, int max_id, int W, int Hh, float half_scale, int min_extent,
                                  const unsigned char* bg_class, int n_class) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= max_id) return;
  int* s = stats + (size_t)id * ST;
  float* bb = bbox + (size_t)id * 4;
  int keep = s[S_CNT] > 0;
  if (keep && bg_class) {
    const int c = s[S_CMIN];
    if (c >= 0 && c < n_class && bg_class[c]) keep = 0;
  }
  const int eu = s[S_UMAX1] - s[S_UMIN], ev = s[S_VMAX1] - s[S_VMIN];
  if (keep && (eu <= min_extent || ev <= min_extent)) keep = 0;
  float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
  if (keep) {
    // int(0.5*scale*(max-min)): torch multiplies the int64 extent by the python float in fp32
    const int mu = (int)__fmul_rn((float)eu, half_scale), mv = (int)__fmul_rn((float)ev, half_scale);
    if (mu == 0 || mv == 0) keep = 0;            // enlarge_bbox returns None (utils.py:42-43)
    else {
      b0 = (float)min(max(s[S_UMIN] - mu, 0), W - 1);  b1 = (float)min(max(s[S_UMAX1] + mu, 0), W - 1);
      b2 = (float)min(max(s[S_VMIN] - mv, 0), Hh - 1); b3 = (float)min(max(s[S_VMAX1] + mv, 0), Hh - 1);
    }
  }
  if (id == 0) { keep = 1; b0 = 0.f; b1 = (float)W; b2 = 0.f; b3 = (float)Hh; }
  s[S_KEEP] = keep;
  bb[0] = b0; bb[1] = b1; bb[2] = b2; bb[3] = b3;
}

// write the frame into a store slot: rgb -> rgbx, depth, and the relabelled instance image
// (dropped instances -> 0 = background, dataset.py:128; -1 stays "unknown")
__global__ void __launch_bounds__(256) k_ingest_write(const int* __restrict__ inst, const unsigned char* __restrict__ rgb,
                                                      const float* __restrict__ depth, const int* __restrict__ stats,
                                                      int max_id, long long n, uchar4* dst_rgbx, float* dst_depth,
                                                      int* dst_inst) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
    const int id = inst[p];
    int out = id;
    if (id >= 0) out = (id < max_id && stats[(size_t)id * ST + S_KEEP]) ? id : 0;
    dst_inst[p] = out;
    if (rgb) dst_rgbx[p] = make_uchar4(rgb[p * 3], rgb[p * 3 + 1], rgb[p * 3 + 2], 0);
    if (depth) dst_depth[p] = depth[p];
  }
}

// ScanNet relabel: the slot's instance image and the per-id tables from K7's output (vmb_assoc_finalize) instead of
// the ingest's.  One grid-stride pass over max(n, max_id): pixel p takes its label (int64 -> int32, -1 stays
// "unknown"); id i < max_id gets keep = the label has a box (abox row i + 1 = label i, column 0) and that box as f32
// (integers below 2^24: exact), every other stats / bbox entry 0.  Ids at or past assoc_max_id have no row: keep 0.
__global__ void __launch_bounds__(256) k_store_relabel(const long long* __restrict__ labels,
                                                       const long long* __restrict__ abox, int assoc_max_id,
                                                       long long n, int max_id, int* dst_inst, int* stats,
                                                       float* bbox) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long m = n > (long long)max_id ? n : (long long)max_id;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < m; p += stride) {
    if (p < n) dst_inst[p] = (int)labels[p];
    if (p < max_id) {
      const long long* r = abox + (p + 1) * 5;
      const int keep = p < assoc_max_id && r[0] != 0;
      int* s = stats + p * ST;
      for (int c = 0; c < ST; ++c) s[c] = 0;
      s[S_KEEP] = keep;
      float* bb = bbox + p * 4;
      for (int c = 0; c < 4; ++c) bb[c] = keep ? (float)r[1 + c] : 0.f;
    }
  }
}

}  // namespace ing
