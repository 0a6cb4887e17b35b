// K7: ScanNet instance association -- utils.box_filter (utils.py:112-208) and the per-label 2-D boxes of
// dataset.py:247-281 on the GPU.  Images are [W][H] (p = u * H + v) as in the FrameStore.
//
//   classify  per-id pixel count / class minimum, 13x13 clipped erosion (= cv2.erode(ones(5,5), iterations=3)),
//             fp64 unprojection without FMA contraction, inclusive oriented-box test against the id's tracked box,
//             per-id counts and the box_filter branch per id; the points to merge are selected and stably sorted by
//             id in row-major (v, u) order (open3d's order on the [H, W] image).
//   voxel     per updated id: its previous cloud followed by the selected points, voxel keys from the id's fp64
//             minimum, a stable sort by (id, key) and one sequential fp64 mean per voxel (open3d VoxelDownSample's
//             summation order), emitted in ascending key order.
//   finalize  label image from the host's final per-id decision and the inside flags, per-label pixel extents
//             (-1 and 0 included), enlarge_bbox in fp64, relabel of "None" boxes to 0.
#pragma once
#include "common.cuh"
#include <limits.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace assoc {

constexpr int NS = 8;     // ints per id in the stats table
enum { S_CNT = 0, S_CMIN = 1, S_FULL = 2, S_ERPX = 3, S_ERPTS = 4, S_INSIDE = 5, S_ACTION = 6, S_VOXELS = 7 };
enum { A_ZERO = 0, A_MERGE = 1, A_NEW = 2, A_NEG = 3 };            // classify's decision (VMB_ASSOC_* in the header)
enum { F_ROW = 1, F_ERODED = 2, F_INSIDE = 4 };
constexpr int BOXW = 16;  // doubles per box row: tracked, center[3], dx[3], dy[3], dz[3], |dx|^2, |dy|^2, |dz|^2
constexpr int RADIUS = 6;
constexpr unsigned long long KEY_NONE = ~0ull;

struct Params {
  int W, H, max_id;
  long long n;
  const int* inst; const int* cls; const float* depth;
  const unsigned char* bg_class; int n_class;
  double fx, fy, cx, cy, P[12];
  int min_pixels;
  double voxel, half_voxel, half_scale;
  const double* boxes;
  const double* pool; const int* cloud_off; const int* cloud_cnt;
  int* stats;
  // scratch
  unsigned char* flags; unsigned char* rowok;
  int* sel_key; int* sel_key_out; int* sel_val; int* sel_val_out;
  int* new_off; int* seg_off;
  double* elem; unsigned long long* ekey; unsigned long long* ekey_out; int* eidx; int* eidx_out; int* head;
  unsigned long long* minb; int* status;
  long long bound;
};

__device__ __forceinline__ unsigned long long ord_key(double x) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(x);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double ord_val(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

__device__ __forceinline__ bool listed(const Params& q, int id) {
  if (id <= 0 || id >= q.max_id) return false;
  const int* s = q.stats + (size_t)id * NS;
  if (s[S_CNT] == 0) return false;
  if (q.bg_class) {
    const int c = s[S_CMIN];
    if (c >= 0 && c < q.n_class && q.bg_class[c]) return false;
  }
  return true;
}

// camera_pose . [(u - cx) z / fx, (v - cy) z / fy, z, 1], rows summed left to right, no contraction
__device__ __forceinline__ void unproject(const Params& q, int u, int v, double z, double* o) {
  const double x = __ddiv_rn(__dmul_rn(__dsub_rn((double)u, q.cx), z), q.fx);
  const double y = __ddiv_rn(__dmul_rn(__dsub_rn((double)v, q.cy), z), q.fy);
#pragma unroll
  for (int r = 0; r < 3; ++r)
    o[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q.P[4 * r], x), __dmul_rn(q.P[4 * r + 1], y)),
                               __dmul_rn(q.P[4 * r + 2], z)), q.P[4 * r + 3]);
}

__device__ __forceinline__ double dot3(const double* a, const double* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

__global__ void k_init(Params q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.max_id) return;
  int* s = q.stats + (size_t)i * NS;
  s[S_CNT] = 0; s[S_CMIN] = INT_MAX; s[S_FULL] = 0; s[S_ERPX] = 0; s[S_ERPTS] = 0; s[S_INSIDE] = 0;
  s[S_ACTION] = A_ZERO; s[S_VOXELS] = 0;
  q.minb[3 * i] = q.minb[3 * i + 1] = q.minb[3 * i + 2] = KEY_NONE;
  if (i == 0) *q.status = 0;
}

// pixel count and class minimum per id (the class decides background, as in the Replica ingest)
__global__ void k_stats(Params q) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < q.n; p += (long long)gridDim.x * blockDim.x) {
    const int id = q.inst[p];
    if (id <= 0 || id >= q.max_id) continue;
    int* s = q.stats + (size_t)id * NS;
    atomicAdd(s + S_CNT, 1);
    if (q.cls) atomicMin(s + S_CMIN, q.cls[p]);
  }
}

// erosion, pass 1: every in-image pixel within RADIUS along u has the same id
__global__ void k_erode_u(Params q) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < q.n; p += (long long)gridDim.x * blockDim.x) {
    const int u = (int)(p / q.H), v = (int)(p - (long long)u * q.H);
    const int id = q.inst[p];
    bool ok = true;
    for (int du = max(u - RADIUS, 0); du <= min(u + RADIUS, q.W - 1); ++du) ok &= q.inst[(long long)du * q.H + v] == id;
    q.rowok[p] = ok;
  }
}

// erosion pass 2 (the column neighbours' rows are uniform AND carry this id) + unprojection + inside test + per-id counts
__global__ void k_classify(Params q) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < q.n; p += (long long)gridDim.x * blockDim.x) {
    const int u = (int)(p / q.H), v = (int)(p - (long long)u * q.H);
    const int id = q.inst[p];
    unsigned char f = 0;
    if (listed(q, id)) {
      bool er = true;
      const long long col = (long long)u * q.H;
      for (int dv = max(v - RADIUS, 0); dv <= min(v + RADIUS, q.H - 1); ++dv)
        er &= q.rowok[col + dv] != 0 && q.inst[col + dv] == id;
      const float d = q.depth[p];
      const bool valid = d > 0.f;
      int* s = q.stats + (size_t)id * NS;
      if (valid) atomicAdd(s + S_FULL, 1);
      if (er) { f |= F_ERODED; atomicAdd(s + S_ERPX, 1); if (valid) atomicAdd(s + S_ERPTS, 1); }
      const double* b = q.boxes + (size_t)id * BOXW;
      if (valid && b[0] != 0.0) {
        double x[3], dd[3];
        unproject(q, u, v, (double)d, x);
        for (int k = 0; k < 3; ++k) dd[k] = __dsub_rn(x[k], b[1 + k]);
        if (fabs(dot3(dd, b + 4)) <= b[13] && fabs(dot3(dd, b + 7)) <= b[14] && fabs(dot3(dd, b + 10)) <= b[15]) {
          f |= F_INSIDE;
          atomicAdd(s + S_INSIDE, 1);
        }
      }
    }
    q.flags[p] = f;
  }
}

// box_filter's branches (utils.py:126-201) for every id
__global__ void k_decide(Params q) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= q.max_id) return;
  int* s = q.stats + (size_t)id * NS;
  int a = A_ZERO;
  if (listed(q, id) && s[S_FULL] > 10) {
    if (q.boxes[(size_t)id * BOXW] != 0.0) a = s[S_INSIDE] >= 1 ? A_MERGE : A_NEG;
    else if (s[S_ERPX] >= q.min_pixels) a = A_NEW;
  }
  s[S_ACTION] = a;
}

// sort keys in row-major (v, u) order: the id of a pixel whose point joins its id's cloud, else max_id (last)
__global__ void k_select(Params q) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < q.n; r += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(r / q.W), u = (int)(r - (long long)v * q.W);
    const long long p = (long long)u * q.H + v;
    const int id = q.inst[p];
    int key = q.max_id;
    if (id > 0 && id < q.max_id) {
      const int a = q.stats[(size_t)id * NS + S_ACTION];
      const unsigned char f = q.flags[p];
      if ((a == A_MERGE && (f & F_INSIDE)) || (a == A_NEW && (f & F_ERODED) && q.depth[p] > 0.f)) key = id;
    }
    q.sel_key[r] = key;
    q.sel_val[r] = (int)r;
  }
}

// per-id segment lengths (old cloud of a merged id + its selected points) and selected-point counts, for the scans
__global__ void k_seg_len(Params q) {
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id > q.max_id) return;
  int nsel = 0, nold = 0;
  if (id < q.max_id) {
    const int* s = q.stats + (size_t)id * NS;
    if (s[S_ACTION] == A_MERGE) { nsel = s[S_INSIDE]; nold = q.cloud_cnt ? q.cloud_cnt[id] : 0; }
    else if (s[S_ACTION] == A_NEW) nsel = s[S_ERPTS];
  }
  q.new_off[id] = nsel;
  q.seg_off[id] = nsel + nold;
}

// element e of the concatenated clouds: its point, the per-id minimum
__global__ void k_elements(Params q) {
  const long long total = q.seg_off[q.max_id];
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < q.bound; e += (long long)gridDim.x * blockDim.x) {
    if (e >= total) { q.ekey[e] = KEY_NONE; q.eidx[e] = (int)e; continue; }
    int lo = 0, hi = q.max_id;                        // last id with seg_off[id] <= e
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (q.seg_off[mid] <= e) lo = mid; else hi = mid; }
    const int id = lo;
    const int seq = (int)(e - q.seg_off[id]);
    const int nold = (q.cloud_cnt && q.stats[(size_t)id * NS + S_ACTION] == A_MERGE) ? q.cloud_cnt[id] : 0;
    double x[3];
    if (seq < nold) {
      const double* src = q.pool + 3 * ((long long)q.cloud_off[id] + seq);
      x[0] = src[0]; x[1] = src[1]; x[2] = src[2];
    } else {
      const int r = q.sel_val_out[q.new_off[id] + seq - nold];
      const int v = r / q.W, u = r - v * q.W;
      unproject(q, u, v, (double)q.depth[(long long)u * q.H + v], x);
    }
    double* o = q.elem + 3 * e;
    for (int k = 0; k < 3; ++k) { o[k] = x[k]; atomicMin(q.minb + 3 * id + k, ord_key(x[k])); }
    q.ekey[e] = (unsigned long long)id;             // the voxel key is filled in by k_keys
    q.eidx[e] = (int)e;
  }
}

// key = id << 48 | kx << 32 | ky << 16 | kz with k = floor((p - (min - voxel / 2)) / voxel)
__global__ void k_keys(Params q) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < q.bound; e += (long long)gridDim.x * blockDim.x) {
    const unsigned long long id = q.ekey[e];
    if (id == KEY_NONE) continue;
    unsigned long long key = id << 48;
    for (int k = 0; k < 3; ++k) {
      const double mb = __dsub_rn(ord_val(q.minb[3 * id + k]), q.half_voxel);
      const double f = floor(__ddiv_rn(__dsub_rn(q.elem[3 * e + k], mb), q.voxel));
      if (!(f >= 0.0 && f < 65536.0)) { atomicOr(q.status, 1); continue; }
      key |= (unsigned long long)f << (16 * (2 - k));
    }
    q.ekey[e] = key;
  }
}

__global__ void k_heads(Params q) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < q.bound; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = q.ekey_out[i];
    q.head[i] = k != KEY_NONE && (i == 0 || q.ekey_out[i - 1] != k);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) q.head[q.bound] = 0;
}

// one sequential fp64 mean per voxel, in input order (the sort is stable); output index = voxel rank
__global__ void k_voxel_mean(Params q, double* out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < q.bound; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = q.ekey_out[i];
    if (k == KEY_NONE || (i > 0 && q.ekey_out[i - 1] == k)) continue;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    long long j = i;
    for (; j < q.bound && q.ekey_out[j] == k; ++j) {
      const double* x = q.elem + 3 * (long long)q.eidx_out[j];
      s0 = __dadd_rn(s0, x[0]); s1 = __dadd_rn(s1, x[1]); s2 = __dadd_rn(s2, x[2]);
    }
    const double c = (double)(j - i);
    double* o = out + 3 * (long long)q.head[i];
    o[0] = __ddiv_rn(s0, c); o[1] = __ddiv_rn(s1, c); o[2] = __ddiv_rn(s2, c);
    atomicAdd(q.stats + (size_t)(k >> 48) * NS + S_VOXELS, 1);
  }
}

// ---- finalize ---------------------------------------------------------------------------------------------------
// final[id]: 0 -> label 0, 1 -> label id (diff pixels -1 when the id merged), 2 -> label -1 (VMB_ASSOC_FINAL_*)
struct FinParams {
  int W, H, max_id; long long n;
  const int* inst; const float* depth; const int* stats; const unsigned char* flags; const int* final_label;
  long long* labels; int* ext; long long* bbox; double half_scale;
};

__global__ void k_fin_init(FinParams q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > q.max_id) return;
  int* e = q.ext + 5 * i;
  e[0] = 0; e[1] = INT_MAX; e[2] = -1; e[3] = INT_MAX; e[4] = -1;
}

__global__ void k_fin_label(FinParams q) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < q.n; p += (long long)gridDim.x * blockDim.x) {
    const int u = (int)(p / q.H), v = (int)(p - (long long)u * q.H);
    const int id = q.inst[p];
    int lab = 0;
    if (id > 0 && id < q.max_id) {
      const int fl = q.final_label[id];
      if (fl == 2) lab = -1;
      else if (fl == 1) {
        lab = id;
        if (q.stats[(size_t)id * NS + S_ACTION] == A_MERGE && q.depth[p] > 0.f && !(q.flags[p] & F_INSIDE)) lab = -1;
      }
    }
    q.labels[p] = lab;
    int* e = q.ext + 5 * (lab + 1);
    atomicAdd(e, 1);
    atomicMin(e + 1, u); atomicMax(e + 2, u); atomicMin(e + 3, v); atomicMax(e + 4, v);
  }
}

// bbox row [present, u_lo, u_hi, v_lo, v_hi] per label + 1: enlarge_bbox with python-int extents, fp64 margins
__global__ void k_fin_box(FinParams q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > q.max_id) return;
  const int* e = q.ext + 5 * i;
  long long* b = q.bbox + 5 * i;
  long long keep = 0, b0 = 0, b1 = 0, b2 = 0, b3 = 0;
  if (e[0] > 0) {
    const int x0 = e[1], x1 = e[2] + 1, y0 = e[3], y1 = e[4] + 1;
    const long long mx = (long long)__dmul_rn(q.half_scale, (double)(x1 - x0));
    const long long my = (long long)__dmul_rn(q.half_scale, (double)(y1 - y0));
    if (mx != 0 && my != 0) {
      keep = 1;
      b0 = min(max(x0 - mx, 0ll), (long long)q.W - 1); b1 = min(max(x1 + mx, 0ll), (long long)q.W - 1);
      b2 = min(max(y0 - my, 0ll), (long long)q.H - 1); b3 = min(max(y1 + my, 0ll), (long long)q.H - 1);
    }
  }
  if (i == 1) { keep = 1; b0 = 0; b1 = q.W; b2 = 0; b3 = q.H; }      // label 0: the full frame (dataset.py:283)
  b[0] = keep; b[1] = b0; b[2] = b1; b[3] = b2; b[4] = b3;
}

// labels whose box is None become background (dataset.py:269-270)
__global__ void k_fin_relabel(FinParams q) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < q.n; p += (long long)gridDim.x * blockDim.x) {
    const long long lab = q.labels[p];
    if (lab != 0 && q.bbox[5 * (lab + 1)] == 0) q.labels[p] = 0;
  }
}

// Handle-owned, grow-only scratch.  The classify outputs (flags, sorted selection) are read by voxel and finalize,
// so the three calls of one frame must use the same handle in order.
struct Workspace {
  DeviceBuffer<unsigned char> pix;      // flags | rowok | sel_key | sel_key_out | sel_val | sel_val_out
  DeviceBuffer<unsigned char> ids;      // new_off | seg_off | minb | status | ext
  DeviceBuffer<unsigned char> el;       // elem | ekey | ekey_out | eidx | eidx_out | head
  DeviceBuffer<void> cub_tmp;
  Params last{};
  bool classified = false;
};

inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }
inline unsigned grid_for(long long n, int bs, int cap) {
  const long long b = (n + bs - 1) / bs;
  return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace assoc
