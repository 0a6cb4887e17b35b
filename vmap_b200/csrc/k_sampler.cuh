// K3: batched depth-guided ray sampler -- one launch for every object of the frame.
// Restates sceneObject.get_training_samples + sample_3d_points + stratified_bins +
// normal_bins_sampling + origin_dirs_W (vmap.py:319-364, 366-459, 45-72, 75-87, 31-41)
// per ray instead of per compacted group, and folds in the stack + /255 of
// train.py:255-260.  No host syncs: the data-dependent max_bound (vmap.py:397) is reduced on
// the device (block reduction + one atomicMax per CTA on an order-preserving key) between the
// two passes, the group branches are per-ray selects.  Both passes run on a (ray chunks x objects)
// grid, so a frame's sampling fills the GPU even with a handful of objects.
//
// Index / bin arithmetic uses explicit round-to-nearest mul/add (no FMA contraction) so
// that with injected randoms the integer outputs and z are bit-identical to torch's
// separate fp32 ops.  Randoms come from Philox4x32-10 unless injected: key (k0, k1) = (low, high 32 bits of seed),
// counter (c0, c1, c2, c3) = (index, stream, object b of the launch, low 32 bits of offset), with
//   stream 0: c0 = keyframe draw f,    word 0 -> kf (only when n_kf <= 2 or f < n_frames - 2)
//   stream 1: c0 = ray i,              words 0, 1 -> u_w, u_h
//   stream 2: c0 = i * 8 + chunk c,    words 0-3 -> u_z[4c .. 4c+3]
//   stream 3: c0 = i * 8 + chunk c,    words 0-3 -> Box-Muller normals 4c .. 4c+3 (this-object rays only)
// so counters are distinct while S <= 32 (c < 8) and N < 2^29 (vmb_sample checks both).  Offsets past 2^32 repeat
// the draws of offset mod 2^32.  The surface sampler of k_eval.cuh draws counter (i, i >> 32, 4, 0): with the same
// seed that is this kernel's stream 0 of object 4 at offset 0, which is harmless (unrelated uses).
// oracle/philox_oracle.py restates
// the draws bit for bit (tests/test_sampler_philox.py, tests/test_sampler_exact_gpu.py).
#pragma once
#include "common.cuh"

struct SampleParams {
  int B, n_frames, n_pix, n1, n2, W, Hh;
  float min_bound, eps, oeps;
  const unsigned char* const* rgbs;
  const float* const* depths;
  const float* const* t_wc;
  const float* const* bbox;
  const int* n_kf;
  const int* latest;
  const float* rays_dir;
  const float* lim;           // [3][33]
  unsigned long long seed, offset;
  const long long* inj_kf; const float* inj_u_w; const float* inj_u_h; const float* inj_u_z; const float* inj_nrm;
  float* pcs; float* z; float* gt_depth; float* gt_colour; unsigned char* rgb_u8;
  unsigned char* sem; unsigned char* mask;
  // shared keyframe store (optional): frames are stored once, objects hold (slot, bbox) tables and the pixel
  // state is derived from the instance image (train.py:126-128: this object -> 1, id -1 -> 2, else 0)
  const uchar4* st_rgbx; const float* st_depth; const int* st_inst; const float* st_twc;
  const int* kf_slot; const float* bbox_flat; const int* obj_id; int kf_stride;
  const unsigned long long* offset_dev;   // optional device-resident draw counter (CUDA-graph replay of a frame)
  int camera_frame;                       // take every keyframe pose as identity: camera-frame points (K11)
  int* kf_out;                            // optional [B][n_frames]: keyframe index of each draw
};

__device__ const float k_identity44[16] = {1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, 1.f};

__device__ __forceinline__ uint32_t sample_offset(const SampleParams& a) {
  return (uint32_t)(a.offset_dev ? *a.offset_dev : a.offset);
}

__device__ __forceinline__ const float* sample_bbox(const SampleParams& a, int b, int kf) {
  return a.st_rgbx ? a.bbox_flat + ((size_t)b * a.kf_stride + kf) * 4 : a.bbox[b] + kf * 4;
}

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t (&out)[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
__device__ __forceinline__ float u01(uint32_t x) { return (float)(x & 0xFFFFFFu) * (1.0f / 16777216.0f); }

struct RayPick { int kf, iw, ih; };

__device__ __forceinline__ RayPick pick_pixel(const SampleParams& a, int b, int i) {
  const int f = i / a.n_pix;
  const int nkf = a.n_kf[b];
  const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32);
  RayPick r;
  if (a.inj_kf) {
    r.kf = (int)a.inj_kf[(size_t)b * a.n_frames + f];
  } else if (nkf > 2 && f >= a.n_frames - 2) {                    // vmap.py:321-331
    r.kf = a.latest[b * 2 + (f - (a.n_frames - 2))];
  } else {
    uint32_t o[4];
    philox4x32_10((uint32_t)f, 0u, (uint32_t)b, sample_offset(a), k0, k1, o);
    r.kf = min((int)(u01(o[0]) * (float)nkf), nkf - 1);
  }
  float uw, uh;
  if (a.inj_u_w) {
    uw = a.inj_u_w[(size_t)b * a.n_frames * a.n_pix + i];
    uh = a.inj_u_h[(size_t)b * a.n_frames * a.n_pix + i];
  } else {
    uint32_t o[4];
    philox4x32_10((uint32_t)i, 1u, (uint32_t)b, sample_offset(a), k0, k1, o);
    uw = u01(o[0]); uh = u01(o[1]);
  }
  const float* bb = sample_bbox(a, b, r.kf);                       // vmap.py:346-351
  r.iw = (int)__fadd_rn(__fmul_rn(uw, __fsub_rn(bb[1], bb[0])), bb[0]);
  r.ih = (int)__fadd_rn(__fmul_rn(uh, __fsub_rn(bb[3], bb[2])), bb[2]);
  r.iw = min(max(r.iw, 0), a.W - 1);
  r.ih = min(max(r.ih, 0), a.Hh - 1);
  return r;
}

// stratified_bins (vmap.py:45-72) for one ray / one bin
__device__ __forceinline__ float strat(float lo, float hi, const float* lim, int n, int k, float u) {
  const float rng = __fsub_rn(hi, lo);
  const float lower = __fadd_rn(__fmul_rn(rng, lim[k]), lo);
  return __fadd_rn(lower, __fmul_rn(u, __fdiv_rn(rng, (float)n)));
}

// order-preserving float <-> uint32 key (atomicMax on the key == max on the float)
__device__ __forceinline__ unsigned int fkey(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Pass 1 (grid = ray chunks x objects): gather pixels, write the 2-D targets, reduce the object's max sampled depth
// (vmap.py:353-354,397) into smax[b] (zeroed by the host before the launch; key 0 is below every float's key).
__global__ void __launch_bounds__(256) k_sample_gather(SampleParams a, unsigned int* __restrict__ smax) {
  const int b = blockIdx.y;
  const int N = a.n_frames * a.n_pix;
  __shared__ float s_max[8];
  const size_t pix_per_kf = (size_t)a.W * a.Hh;
  float mx = -3.0e38f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    const RayPick r = pick_pixel(a, b, i);
    if (a.kf_out && i % a.n_pix == 0) a.kf_out[(size_t)b * a.n_frames + i / a.n_pix] = r.kf;
    uchar4 px;
    float d;
    if (a.st_rgbx) {
      const size_t pi = (size_t)a.kf_slot[(size_t)b * a.kf_stride + r.kf] * pix_per_kf + (size_t)r.iw * a.Hh + r.ih;
      px = a.st_rgbx[pi];
      d = a.st_depth[pi];
      const int id = a.st_inst[pi];
      px.w = id == a.obj_id[b] ? 1 : (id == -1 ? 2 : 0);
    } else {
      const size_t pi = (size_t)r.kf * pix_per_kf + (size_t)r.iw * a.Hh + r.ih;
      px = reinterpret_cast<const uchar4*>(a.rgbs[b])[pi];
      d = a.depths[b][pi];
    }
    const size_t o = (size_t)b * N + i;
    a.gt_depth[o] = d;
    a.gt_colour[o * 3 + 0] = (float)px.x / 255.f;                 // train.py:257
    a.gt_colour[o * 3 + 1] = (float)px.y / 255.f;
    a.gt_colour[o * 3 + 2] = (float)px.z / 255.f;
    if (a.rgb_u8) { a.rgb_u8[o * 3] = px.x; a.rgb_u8[o * 3 + 1] = px.y; a.rgb_u8[o * 3 + 2] = px.z; }
    a.sem[o] = px.w;
    a.mask[o] = !(d <= a.min_bound);                              // vmap.py:395,407
    mx = fmaxf(mx, d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = s_max[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, s_max[w]);
    atomicMax(smax + b, fkey(m));
  }
}

// Pass 2 (grid = ray chunks x objects): per-ray sample depths and 3-D points (vmap.py:366-459)
// N1 / N2 > 0: compile-time bin counts (the shipped object (1, 9) and background (5, 9) configurations): every loop
// unrolls and the per-ray random / normal arrays live in registers; 0 = run-time counts (arrays in local memory).
template <int N1, int N2>
__global__ void __launch_bounds__(256) k_sample_points(SampleParams a, const unsigned int* __restrict__ smax) {
  const int b = blockIdx.y;
  const int N = a.n_frames * a.n_pix;
  const int n1 = N1 ? N1 : a.n1, n2 = N2 ? N2 : a.n2;
  const int S = n1 + n2;
  constexpr int SMAX = (N1 && N2) ? N1 + N2 : 32, N2MAX = N2 ? N2 : 32;
  const float max_bound = fkey_inv(smax[b]);
  // a thread owns a ray (S x 16 B of output), so direct stores would touch 32 lines per instruction: the block's
  // rays are consecutive in memory, results are staged in shared memory and written out as one coalesced span
  extern __shared__ float s_out[];                 // [256][S] z | [256][S][3] points
  float* s_z = s_out;
  float* s_p = s_out + 256 * S;

  const float* limS = a.lim, * lim1 = a.lim + 33, * lim2 = a.lim + 66;
  const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32);
  for (int base = blockIdx.x * 256; base < N; base += gridDim.x * 256) {
    const int i = base + threadIdx.x;
    if (i < N) {
    const RayPick r = pick_pixel(a, b, i);
    const size_t o = (size_t)b * N + i;
    const float d = a.gt_depth[o];
    const int state = a.sem[o];
    const bool invalid = d <= a.min_bound;
    const bool this_obj = (state == 1) && !invalid;

    float uz[SMAX], nz[N2MAX];
    if (a.inj_u_z) {
#pragma unroll
      for (int s = 0; s < S; ++s) uz[s] = a.inj_u_z[o * S + s];
    } else {
#pragma unroll
      for (int c = 0; c * 4 < S; ++c) {
        uint32_t q[4];
        philox4x32_10((uint32_t)i * 8u + c, 2u, (uint32_t)b, sample_offset(a), k0, k1, q);
#pragma unroll
        for (int j = 0; j < 4; ++j) if (c * 4 + j < S) uz[c * 4 + j] = u01(q[j]);
      }
    }
    if (this_obj) {
      if (a.inj_nrm) {
#pragma unroll
        for (int s = 0; s < n2; ++s) nz[s] = a.inj_nrm[o * n2 + s];
      } else {
        const float sd = a.eps / 3.0f;                            // vmap.py:432 delta/3
#pragma unroll
        for (int c = 0; c * 4 < n2; ++c) {
          uint32_t q[4];
          philox4x32_10((uint32_t)i * 8u + c, 3u, (uint32_t)b, sample_offset(a), k0, k1, q);
          const float r0 = sqrtf(-2.f * logf(1.f - u01(q[0]))), r1 = sqrtf(-2.f * logf(1.f - u01(q[2])));
          float s0, c0, s1, c1;
          sincospif(2.f * u01(q[1]), &s0, &c0);
          sincospif(2.f * u01(q[3]), &s1, &c1);
          const float g[4] = {r0 * c0, r0 * s0, r1 * c1, r1 * s1};
#pragma unroll
          for (int j = 0; j < 4; ++j) if (c * 4 + j < n2) nz[c * 4 + j] = g[j] * sd;
        }
      }
      if (N2) {                                                   // .sort() (vmap.py:81): odd-even transposition network,
#pragma unroll                                                    // static indices only (registers)
        for (int round = 0; round < N2MAX; ++round) {
#pragma unroll
          for (int x = round & 1; x + 1 < N2MAX; x += 2) {
            const float lo = fminf(nz[x], nz[x + 1]), hi = fmaxf(nz[x], nz[x + 1]);
            nz[x] = lo; nz[x + 1] = hi;
          }
        }
      } else {
        for (int x = 1; x < n2; ++x) {                            // insertion sort
          const float v = nz[x];
          int y = x - 1;
          while (y >= 0 && nz[y] > v) { nz[y + 1] = nz[y]; --y; }
          nz[y + 1] = v;
        }
      }
    }

    const float* dc = a.rays_dir + ((size_t)r.iw * a.Hh + r.ih) * 3;   // vmap.py:357
    const float* T = a.camera_frame ? k_identity44
                   : a.st_rgbx ? a.st_twc + (size_t)a.kf_slot[(size_t)b * a.kf_stride + r.kf] * 16
                               : a.t_wc[b] + r.kf * 16;                // vmap.py:360
    const float dw0 = fmaf(T[2], dc[2], fmaf(T[1], dc[1], T[0] * dc[0]));      // vmap.py:37
    const float dw1 = fmaf(T[6], dc[2], fmaf(T[5], dc[1], T[4] * dc[0]));
    const float dw2 = fmaf(T[10], dc[2], fmaf(T[9], dc[1], T[8] * dc[0]));
    const float o0 = T[3], o1 = T[7], o2 = T[11];                              // vmap.py:39

#pragma unroll
    for (int s = 0; s < S; ++s) {
      float zz;
      if (invalid) {
        zz = strat(a.min_bound, max_bound, limS, S, s, uz[s]);                 // vmap.py:400-404
      } else if (s < n1) {
        zz = strat(a.min_bound, __fsub_rn(d, a.eps), lim1, n1, s, uz[s]);    // vmap.py:413-415
      } else if (this_obj) {
        const float bn = fminf(fmaxf(nz[s < n1 ? 0 : s - n1], -a.eps), a.eps);            // vmap.py:82
        zz = __fadd_rn(d, bn);                                                 // vmap.py:83
      } else {
        zz = strat(__fsub_rn(d, a.eps), __fadd_rn(d, a.oeps), lim2, n2, s - n1, uz[s]);   // vmap.py:447-450
      }
      s_z[threadIdx.x * S + s] = zz;
      float* pc = s_p + (threadIdx.x * S + s) * 3;                             // vmap.py:455
      pc[0] = __fadd_rn(o0, __fmul_rn(dw0, zz));
      pc[1] = __fadd_rn(o1, __fmul_rn(dw1, zz));
      pc[2] = __fadd_rn(o2, __fmul_rn(dw2, zz));
    }
    }
    __syncthreads();
    const int nv = min(256, N - base);
    float* gz = a.z + ((size_t)b * N + base) * S;
    for (int k = threadIdx.x; k < nv * S; k += 256) gz[k] = s_z[k];
    float* gp = a.pcs + ((size_t)b * N + base) * S * 3;
    for (int k = threadIdx.x; k < nv * S * 3; k += 256) gp[k] = s_p[k];
    __syncthreads();
  }
}
