// Layer-wise tensor-core path for wide models (hidden 64 / 128 / 256: the separate background model
// and the iMAP whole-scene model).  One object's weights (up to 640 KB of fp16) and a tile's
// activations no longer fit in shared memory together, so each layer runs as a wgmma GEMM
// (k_gemm_umma.cuh) over ALL points of the object, activations living in an L2-resident workspace;
// the thin stages between the GEMMs (positional embedding, heads, volume render + loss, head
// gradients, PE gradient) are small CUDA-core kernels.  Same arithmetic and the same reference lines
// as k_step_fp32.cuh / k_step_fused.cuh: embedding.py:82-91, model.py:54-85, render_rays.py:4-96,
// loss.py:5-62 and their backward.
// The pose step (k_track_lw.cuh) runs the same network through the pieces written here once: the embedding block
// (pe_block), a warp's head rows (HeadRows: staging, the heads, the dYc gate) and the GEMM chains (forward_gemms,
// InputGrads).  Each step keeps its own render and loss.
//
// Workspace row layouts (fp16 unless noted), P = R*S points of the object:
//   E  [P][144]: cols 0..86 = emb[0..86] (xyz/scale, sin k=0..3), 87 = 1, 88..95 = 0,
//                cols 96..137 = emb[87..128] (sin k=4,5), 138 = 1, 139..143 = 0
//                (the constant-1 columns make three bias gradients fall out of the wgrad GEMMs)
//   X1..X4, XC [P][H] activations;  dYa, dYb, dYc [P][H] (loss-scaled by 2^8);  dE [P][144] fp32
// Weight image (per object, written by the fused AdamW): row-major fp16
//   W_in [H][96] | W_m1 [H][H] | W_cat [H][H+96] | W_m2 [H][H] | W_cl [H][H+48]   (zero under pad / ones columns)
#pragma once
#include <string>
#include <type_traits>
#include "common.cuh"
#include "k_step_fp32.cuh"
#include "k_gemm_umma.cuh"

namespace lw {

constexpr int EW = 144;          // embedding row width
constexpr int E1W = 96, E2W = 48, ONES1 = 87, ONES2 = 42;

__host__ __device__ inline long long img_halves(int H) { return (long long)H * (4 * H + 240); }
__host__ __device__ inline long long off_m1(int H) { return 96LL * H; }
__host__ __device__ inline long long off_cat(int H) { return off_m1(H) + (long long)H * H; }
__host__ __device__ inline long long off_m2(int H) { return off_cat(H) + (long long)H * (H + 96); }
__host__ __device__ inline long long off_cl(int H) { return off_m2(H) + (long long)H * H; }

// param index -> half index inside the wide-model image (or -1)
static void fill_image_index(const VmbLayout& L, int* idx) {
  const int H = L.H;
  for (int i = 0; i < L.P; ++i) idx[i] = -1;
  for (int o = 0; o < H; ++o) {
    for (int j = 0; j < VMB_E1; ++j) idx[L.o_Win + o * VMB_E1 + j] = (int)((long long)o * 96 + j);
    for (int k = 0; k < H; ++k) idx[L.o_Wm1 + o * H + k] = (int)(off_m1(H) + (long long)o * H + k);
    for (int k = 0; k < H + VMB_E1; ++k) idx[L.o_Wcat + o * (H + VMB_E1) + k] = (int)(off_cat(H) + (long long)o * (H + 96) + k);
    for (int k = 0; k < H; ++k) idx[L.o_Wm2 + o * H + k] = (int)(off_m2(H) + (long long)o * H + k);
    for (int k = 0; k < H + L.e2; ++k) idx[L.o_Wcl + o * (H + L.e2) + k] = (int)(off_cl(H) + (long long)o * (H + 48) + k);
  }
}

// point counts of the workspaces' per-point buffers are rounded up to whole 128-point blocks
inline long long pad_points(long long P) { return (P + 127) / 128 * 128; }

struct Workspace {
  DeviceBuffer<__half> E, X1, X2, X3, X4, XC, dYa, dYb, dYc, dh16;
  DeviceBuffer<float> dalpha_s, dE;
  // side stream of the backward pass: the weight-gradient GEMMs of a layer depend only on that layer's dY, so they run
  // beside the input-gradient chain (fork / join with events; inside a stream capture they become parallel graph branches)
  cudaStream_t side = nullptr;
  cudaEvent_t ev_main[5] = {}, ev_side[2] = {};
  cudaError_t ensure_streams() {
    if (side) return cudaSuccess;
    cudaError_t e = cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
    for (auto& v : ev_main) if (e == cudaSuccess) e = cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    for (auto& v : ev_side) if (e == cudaSuccess) e = cudaEventCreateWithFlags(&v, cudaEventDisableTiming);
    return e;
  }
  ~Workspace() {
    for (auto v : ev_main) if (v) cudaEventDestroy(v);
    for (auto v : ev_side) if (v) cudaEventDestroy(v);
    if (side) cudaStreamDestroy(side);
  }
  // every buffer for P points of a hidden-H model
  cudaError_t grow(long long P, int H, bool capturing) {
    const size_t Pp = (size_t)pad_points(P);
    cudaError_t e = E.grow(Pp * EW * 2, capturing);
    for (auto* x : {&X1, &X2, &X3, &X4, &XC, &dYa, &dYb, &dYc})
      if (e == cudaSuccess) e = x->grow(Pp * H * 2, capturing);
    if (e == cudaSuccess) e = dh16.grow(Pp * 8 * 2, capturing);
    if (e == cudaSuccess) e = dalpha_s.grow(Pp * 4, capturing);
    if (e == cudaSuccess) e = dE.grow(Pp * EW * 4, capturing);
    return e;
  }
};

// sin / cos of pi 2^k x by one MUFU pair + angle doubling
__device__ __forceinline__ void sincos_ladder6(float proj, float (&s)[6], float (&c)[6]) {
  const float r = proj - 2.0f * rintf(0.5f * proj);
  s[0] = __sinf(VMB_PI_F * r);
  c[0] = __cosf(VMB_PI_F * r);
#pragma unroll
  for (int k = 1; k < 6; ++k) {
    const float s2 = s[k - 1] + s[k - 1];
    s[k] = s2 * c[k - 1];
    c[k] = fmaf(-s2, s[k - 1], 1.0f);
  }
}

// ---------------------------------------------------------------------------------------------
// positional embedding: 128 points per block, rows assembled in shared memory, written coalesced
// ---------------------------------------------------------------------------------------------
// The E rows (EW halves each) of this block's 128 points of P, this thread's at the network input t (p / scale, or the
// posed point of k_tlw_pe): xyz, the sin bands, the constant-1 and zero columns
__device__ __forceinline__ void pe_block(float t0, float t1, float t2, const float* __restrict__ dirs, long long P,
                                         __half* __restrict__ E) {
  __shared__ __align__(16) __half row[128 * EW];
  __half* r = row + threadIdx.x * EW;
  r[0] = __float2half_rn(t0); r[1] = __float2half_rn(t1); r[2] = __float2half_rn(t2);
  for (int d = 0; d < VMB_NDIRS; ++d) {
    float s[6], c[6];
    sincos_ladder6(fmaf(__ldg(dirs + d * 3 + 2), t2, fmaf(__ldg(dirs + d * 3 + 1), t1, __ldg(dirs + d * 3) * t0)), s, c);
#pragma unroll
    for (int k = 0; k < 4; ++k) r[3 + k * VMB_NDIRS + d] = __float2half_rn(s[k]);
    r[E1W + d] = __float2half_rn(s[4]);
    r[E1W + VMB_NDIRS + d] = __float2half_rn(s[5]);
  }
  r[ONES1] = __float2half_rn(1.0f);
  for (int j = ONES1 + 1; j < E1W; ++j) r[j] = __float2half_rn(0.f);
  r[E1W + ONES2] = __float2half_rn(1.0f);
  for (int j = E1W + ONES2 + 1; j < EW; ++j) r[j] = __float2half_rn(0.f);
  __syncthreads();
  // 128 rows x 288 B are contiguous in E
  const long long p0 = (long long)blockIdx.x * 128;
  const uint4* src = reinterpret_cast<const uint4*>(row);
  uint4* dst = reinterpret_cast<uint4*>(E + p0 * EW);
  const long long n16 = min(128LL, P - p0) * (EW * 2 / 16);
  for (long long i = threadIdx.x; i < n16; i += 128) dst[i] = src[i];
}

__global__ void __launch_bounds__(128) k_lw_pe(const float* __restrict__ pcs, const float* __restrict__ dirs,
                                               const float* __restrict__ scale_ptr, long long P, __half* __restrict__ E) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const float scale = *scale_ptr;
  const long long p = (long long)blockIdx.x * 128 + threadIdx.x;
  float t0 = 0.f, t1 = 0.f, t2 = 0.f;
  if (p < P) { t0 = pcs[p * 3] / scale; t1 = pcs[p * 3 + 1] / scale; t2 = pcs[p * 3 + 2] / scale; }
  pe_block(t0, t1, t2, dirs, P, E);
}

// ---------------------------------------------------------------------------------------------
// heads: alpha = (w_a . fc4 + b_a) * 10 -> occupancy; colour = sigmoid(W_oc hc + b_oc)   (model.py:71-83)
// ---------------------------------------------------------------------------------------------
template <int H>
__global__ void __launch_bounds__(128) k_lw_heads(const __half* __restrict__ X4, const __half* __restrict__ XC,
                                                  const float* __restrict__ P, VmbLayout L, long long np,
                                                  float* __restrict__ occ, float* __restrict__ col, int raw) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  // raw != 0 (eval_points, trainer.py:77-90): occ receives alpha*10 before the sigmoid
  __shared__ float w[4 * H];
  for (int i = threadIdx.x; i < H; i += 128) w[i] = P[L.o_Wa + i];
  for (int i = threadIdx.x; i < 3 * H; i += 128) w[H + i] = P[L.o_Woc + i];
  __syncthreads();
  const long long p = (long long)blockIdx.x * 128 + threadIdx.x;
  if (p >= np) return;
  float a = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
  const uint4* x4 = reinterpret_cast<const uint4*>(X4 + p * H);
  const uint4* xc = reinterpret_cast<const uint4*>(XC + p * H);
#pragma unroll 4
  for (int q = 0; q < H / 8; ++q) {
    const uint4 u = x4[q], v = xc[q];
    const __half* hu = reinterpret_cast<const __half*>(&u);
    const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f4 = __half2float(hu[j]), fc = __half2float(hv[j]);
      const int o = q * 8 + j;
      a = fmaf(f4, w[o], a);
      c0 = fmaf(fc, w[H + o], c0); c1 = fmaf(fc, w[2 * H + o], c1); c2 = fmaf(fc, w[3 * H + o], c2);
    }
  }
  occ[p] = raw ? (a + P[L.o_ba]) * 10.0f : vmb_sigmoid((a + P[L.o_ba]) * 10.0f);
  col[p * 3] = vmb_sigmoid(c0 + P[L.o_boc]); col[p * 3 + 1] = vmb_sigmoid(c1 + P[L.o_boc + 1]);
  col[p * 3 + 2] = vmb_sigmoid(c2 + P[L.o_boc + 2]);
}

// ---------------------------------------------------------------------------------------------
// volume render + losses + d(loss)/d(raw alpha, raw colour): one thread per ray
// (render_rays.py:4-8,26-34,47-96; loss.py:5-62) -- same code path as k_step_fp32 phase C
// ---------------------------------------------------------------------------------------------
struct RenderArgs {
  int b, R, S, B;
  const float* z; const float* gt_depth; const float* gt_colour; const unsigned char* sem; const unsigned char* mask;
  const int* counts; float cs, os; int backward;
  float* loss_terms; float* r_depth; float* r_var; float* r_colour; float* r_opacity;
};
template <int H> constexpr int hr_pitch() { return H * 2 + 16; }
template <int H> constexpr int hr_smem() { return 4 * 32 * hr_pitch<H>(); }         // 4 warps x 32 rows (fc4, then hc)
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ptx::smem_u32(dst)), "l"(src) : "memory");
}
// One warp's ray in the heads / render kernels (k_lw_heads_render, k_tlw_render), lane = sample: the heads forward on
// the staged fc4 / hc rows and the head backward into dY_c.  A warp stages its ray's fc4 rows, then its hc rows, in ONE
// shared-memory buffer with coalesced 16 B asynchronous copies (a lane walking its own 2H-byte row straight from global
// memory is a chain of dependent L2 round trips); the row pitch of 2H + 16 B makes the per-lane 16 B reads
// conflict-free, and one buffer per warp keeps three blocks resident per SM at H = 256 so the copies of one warp hide
// behind the arithmetic of the others.
template <int H>
struct HeadRows {
  static constexpr int PITCH = hr_pitch<H>(), LPR = H / 8, RPP = 32 / LPR;      // lanes per row, rows per copy pass
  float* w;                 // the block's head weights in shared memory: [0,H) out_alpha row, [H,4H) out_color rows
  unsigned char* srow;      // this warp's 32 rows
  int lane, S;

  // every thread of the block; the caller synchronises before the first read
  __device__ __forceinline__ void load(const float* __restrict__ P, const VmbLayout& L) {
    for (int i = threadIdx.x; i < H; i += 128) w[i] = P[L.o_Wa + i];
    for (int i = threadIdx.x; i < 3 * H; i += 128) w[H + i] = P[L.o_Woc + i];
  }
  __device__ __forceinline__ uint4* row() const { return reinterpret_cast<uint4*>(srow + lane * PITCH); }
  // the ray's S rows [pb, pb + S) of X, once the rows staged before are no longer read
  __device__ __forceinline__ void stage(const __half* X, long long pb) {
    __syncwarp();
#pragma unroll 4
    for (int r0 = 0; r0 < S; r0 += RPP) {
      const int r = r0 + lane / LPR, cq = lane % LPR;
      if (r < S) cp_async16(srow + r * PITCH + cq * 16, X + (pb + r) * H + cq * 8);
    }
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    __syncwarp();
  }
  // w_a . fc4 of the staged fc4 row, in two chains: the dot product is FMA-latency bound otherwise
  __device__ __forceinline__ float alpha() const {
    const uint4* xrow = row();
    float ha = 0.f, hb = 0.f;
#pragma unroll 4
    for (int q = 0; q < H / 8; ++q) {
      const uint4 u = xrow[q];
      const __half* hu = reinterpret_cast<const __half*>(&u);
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        ha = fmaf(__half2float(hu[j]), w[q * 8 + j], ha);
        hb = fmaf(__half2float(hu[j + 1]), w[q * 8 + j + 1], hb);
      }
    }
    return ha + hb;
  }
  // W_oc hc of the staged hc row
  __device__ __forceinline__ void colour(float& h0, float& h1, float& h2) const {
    const uint4* xrow = row();
    h0 = h1 = h2 = 0.f;
#pragma unroll 4
    for (int q = 0; q < H / 8; ++q) {
      const uint4 v = xrow[q];
      const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float fc = __half2float(hv[j]);
        const int o = q * 8 + j;
        h0 = fmaf(fc, w[H + o], h0); h1 = fmaf(fc, w[2 * H + o], h1); h2 = fmaf(fc, w[3 * H + o], h2);
      }
    }
  }
  // The staged hc row gated IN PLACE into dY_c = relu'(hc) * (d @ W_oc), clamped to the fp16 range +-60000, from the
  // loss-scaled d(raw colour) d0..d2.  Returns how many values pass 60000: the clamped dY_c elements, and the elements
  // where dY4's rank-1 term da w_a (da the loss-scaled d(raw alpha)) does on its own.
  __device__ __forceinline__ int gate(float d0, float d1, float d2, float da) {
    uint4* xc = row();
    int n = 0;
#pragma unroll 4
    for (int q = 0; q < H / 8; ++q) {
      const uint4 v = xc[q];
      const __half* hv = reinterpret_cast<const __half*>(&v);
      uint32_t r[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int o = q * 8 + 2 * j;
        float x0 = fmaf(d2, w[3 * H + o], fmaf(d1, w[2 * H + o], d0 * w[H + o]));
        float x1 = fmaf(d2, w[3 * H + o + 1], fmaf(d1, w[2 * H + o + 1], d0 * w[H + o + 1]));
        const bool g0 = __half2float(hv[2 * j]) > 0.f, g1 = __half2float(hv[2 * j + 1]) > 0.f;
        n += (g0 && fabsf(x0) > 60000.f) + (g1 && fabsf(x1) > 60000.f);
        n += (fabsf(da * w[o]) > 60000.f) + (fabsf(da * w[o + 1]) > 60000.f);
        x0 = g0 ? fminf(fmaxf(x0, -60000.f), 60000.f) : 0.f;
        x1 = g1 ? fminf(fmaxf(x1, -60000.f), 60000.f) : 0.f;
        __half2 hh = __floats2half2_rn(x0, x1);
        r[j] = *reinterpret_cast<uint32_t*>(&hh);
      }
      xc[q] = make_uint4(r[0], r[1], r[2], r[3]);
    }
    return n;
  }
  // the ray's dY_c rows out as whole 2H-byte rows (the mirror image of stage), once every lane has gated its row
  __device__ __forceinline__ void store(__half* __restrict__ dYc, long long pb) const {
    __syncwarp();
#pragma unroll 4
    for (int r0 = 0; r0 < S; r0 += RPP) {
      const int r = r0 + lane / LPR, cq = lane % LPR;
      if (r < S) *reinterpret_cast<uint4*>(dYc + (pb + r) * H + cq * 8) = *reinterpret_cast<const uint4*>(srow + r * PITCH + cq * 16);
    }
  }
};

// Heads + render + loss + head gradients in ONE kernel, one warp per ray, lane = sample (n_samples <= 32):
//   forward   alpha / colour heads of the lane's point (the fc4 / hc rows are read once),
//   render    transmittance as a warp product scan, the ray sums as warp reductions,
//   backward  d(occupancy, colour) with the suffix sum as a warp scan, then dYc = relu'(hc) * (d_rawc @ W_oc)
//             (fp16, x2^8), the scaled copies of d_alpha for the rank-1 term / the head wgrad GEMMs, and the bias
//             gradients of the two heads.
// Replaces three launches (heads, render, head gradients) and the round trip of occupancy / colour / dhead through HBM.
template <int H>
__global__ void __launch_bounds__(128) k_lw_heads_render(RenderArgs a, const __half* __restrict__ X4, const __half* __restrict__ XC,
                                                         const float* __restrict__ P, VmbLayout L, __half* __restrict__ dYc,
                                                         __half* __restrict__ dh16, float* __restrict__ dalpha_s,
                                                         float* __restrict__ G) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  extern __shared__ __align__(16) unsigned char hr_rows[];
  __shared__ float w[4 * H];
  __shared__ int s_on[3];
  __shared__ float s_loss[3], s_b[4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, S = a.S, b = a.b;
  HeadRows<H> hr{w, hr_rows + warp * (32 * HeadRows<H>::PITCH), lane, S};
  hr.load(P, L);
  if (threadIdx.x < 3) {
    int on = 1;
    for (int i = 0; i < a.B; ++i) on &= (a.counts[i * 4 + threadIdx.x] != 0);
    s_on[threadIdx.x] = on; s_loss[threadIdx.x] = 0.f;
  }
  if (threadIdx.x < 4) s_b[threadIdx.x] = 0.f;
  __syncthreads();
  const unsigned FULL = 0xffffffffu;
  const float b_a = P[L.o_ba], b_c0 = P[L.o_boc], b_c1 = P[L.o_boc + 1], b_c2 = P[L.o_boc + 2];
  const float inv_nd = 1.f / ((float)a.counts[b * 4 + 0] + 1e-10f);
  const float inv_no = 1.f / ((float)a.counts[b * 4 + 1] + 1e-10f);
  const float inv_ns = 1.f / ((float)a.counts[b * 4 + 2] + 1e-10f);
  const float on_d = s_on[0] ? 1.f : 0.f, on_c = s_on[1] ? 1.f : 0.f, on_o = s_on[2] ? 1.f : 0.f;
  const bool in = lane < S;
  float l_d = 0.f, l_c = 0.f, l_o = 0.f;              // every lane carries the same per-ray values; lane 0's are used
  float sb0 = 0.f, sb1 = 0.f, sb2 = 0.f, sb3 = 0.f;   // this lane's share of the head bias gradients
  for (int ray = blockIdx.x * 4 + warp; ray < a.R; ray += gridDim.x * 4) {
    const long long pb = (long long)ray * S, pi = pb + lane;
    hr.stage(X4, pb);
    float ha = 0.f, h0 = 0.f, h1 = 0.f, h2 = 0.f;
    if (in) ha = hr.alpha();
    hr.stage(XC, pb);                                 // hc stays staged for the backward half
    float oc = 0.f, zz = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
    if (in) {
      hr.colour(h0, h1, h2);
      oc = vmb_sigmoid((ha + b_a) * 10.0f);
      c0 = vmb_sigmoid(h0 + b_c0); c1 = vmb_sigmoid(h1 + b_c1); c2 = vmb_sigmoid(h2 + b_c2);
      zz = a.z[pi];
    }
    const float om = 1.f - oc + 1e-10f;               // lanes past the ray: 1
    float incl = om;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const float t = __shfl_up_sync(FULL, incl, d); if (lane >= d) incl *= t; }
    float T = __shfl_up_sync(FULL, incl, 1);
    if (lane == 0) T = 1.f;
    const float wgt = oc * T;
    const float D = warp_sum(wgt * zz), O = warp_sum(wgt), C0 = warp_sum(wgt * c0), C1 = warp_sum(wgt * c1), C2 = warp_sum(wgt * c2);
    const float dz = zz - D;
    const float V = warp_sum(wgt * dz * dz);
    if (lane == 0) {
      if (a.r_depth) a.r_depth[(size_t)b * a.R + ray] = D;
      if (a.r_var) a.r_var[(size_t)b * a.R + ray] = V;
      if (a.r_opacity) a.r_opacity[(size_t)b * a.R + ray] = O;
      if (a.r_colour) { float* rc = a.r_colour + ((size_t)b * a.R + ray) * 3; rc[0] = C0; rc[1] = C1; rc[2] = C2; }
    }
    const int sv = a.sem[ray];
    const float m_o = (sv != 0) ? 1.f : 0.f, m_s = (sv != 2) ? 1.f : 0.f, m_d = (a.mask[ray] != 0) ? m_o : 0.f;
    const float gd = a.gt_depth[ray];
    const float* gc = a.gt_colour + (size_t)ray * 3;
    const float info = 1.f / (sqrtf(V) + 1e-4f);
    const float e_d = D - gd, e_o = O - m_o, e_c0 = C0 - gc[0], e_c1 = C1 - gc[1], e_c2 = C2 - gc[2];
    l_d += on_d * fabsf(e_d) * m_d * info * inv_nd;
    l_c += on_c * (fabsf(e_c0) + fabsf(e_c1) + fabsf(e_c2)) * m_o * inv_no;
    l_o += on_o * fabsf(e_o) * m_s * inv_ns;
    if (!a.backward) continue;
    const float gD = on_d * vmb_sign(e_d) * m_d * info * inv_nd;
    const float kc = on_c * a.cs * m_o * inv_no;
    const float gC0 = kc * vmb_sign(e_c0), gC1 = kc * vmb_sign(e_c1), gC2 = kc * vmb_sign(e_c2);
    const float gO = on_o * a.os * vmb_sign(e_o) * m_s * inv_ns;
    const float Gs = fmaf(gD, zz, fmaf(gC0, c0, fmaf(gC1, c1, fmaf(gC2, c2, gO))));
    float sfx = Gs * wgt;                             // inclusive suffix sum of G_j w_j, then shifted to exclusive
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const float t = __shfl_down_sync(FULL, sfx, d); if (lane + d < 32) sfx += t; }
    float suffix = __shfl_down_sync(FULL, sfx, 1);
    if (lane == 31) suffix = 0.f;
    if (in) {
      const float docc = Gs * T - suffix / om;
      float4 dh;                                      // d(loss) / d(raw alpha, raw colour) of this point
      dh.x = 10.0f * docc * oc * (1.f - oc);
      dh.y = gC0 * wgt * c0 * (1.f - c0); dh.z = gC1 * wgt * c1 * (1.f - c1); dh.w = gC2 * wgt * c2 * (1.f - c2);
      sb0 += dh.x; sb1 += dh.y; sb2 += dh.z; sb3 += dh.w;
      dalpha_s[pi] = LS * dh.x;
      __half2 h01 = __floats2half2_rn(fminf(fmaxf(LS * dh.x, -60000.f), 60000.f), fminf(fmaxf(LS * dh.y, -60000.f), 60000.f));
      __half2 h23 = __floats2half2_rn(fminf(fmaxf(LS * dh.z, -60000.f), 60000.f), fminf(fmaxf(LS * dh.w, -60000.f), 60000.f));
      reinterpret_cast<uint4*>(dh16)[pi] = make_uint4(*reinterpret_cast<uint32_t*>(&h01), *reinterpret_cast<uint32_t*>(&h23), 0u, 0u);
      hr.gate(LS * dh.y, LS * dh.z, LS * dh.w, LS * dh.x);     // the clamp count is the pose step's
    }
    hr.store(dYc, pb);
  }
  if (lane == 0) { atomicAdd(&s_loss[0], l_d); atomicAdd(&s_loss[1], l_c); atomicAdd(&s_loss[2], l_o); }
  if (a.backward) {
    sb0 = warp_sum(sb0); sb1 = warp_sum(sb1); sb2 = warp_sum(sb2); sb3 = warp_sum(sb3);
    if (lane == 0) { atomicAdd(&s_b[0], sb0); atomicAdd(&s_b[1], sb1); atomicAdd(&s_b[2], sb2); atomicAdd(&s_b[3], sb3); }
  }
  __syncthreads();
  if (threadIdx.x < 3 && a.loss_terms) atomicAdd(a.loss_terms + b * 4 + threadIdx.x, s_loss[threadIdx.x]);
  if (threadIdx.x == 3 && a.loss_terms) atomicAdd(a.loss_terms + b * 4 + 3, s_loss[0] + a.cs * s_loss[1] + a.os * s_loss[2]);
  if (a.backward && G) {
    if (threadIdx.x == 32) atomicAdd(G + L.o_ba, s_b[0]);
    if (threadIdx.x >= 33 && threadIdx.x < 36) atomicAdd(G + L.o_boc + threadIdx.x - 33, s_b[threadIdx.x - 32]);
  }
}

// column sums of a [P][H] fp16 gradient block -> bias gradient (x 2^-8); `rows` rows per block
__global__ void __launch_bounds__(256) k_lw_colsum(const __half* __restrict__ dY, long long np, int H, int rows, float* __restrict__ gb) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const int c = threadIdx.x;
  if (c >= H) return;
  const long long r0 = (long long)blockIdx.x * rows, r1 = min(np, r0 + rows);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  long long r = r0;
  for (; r + 3 < r1; r += 4) {
    s0 += __half2float(dY[r * H + c]); s1 += __half2float(dY[(r + 1) * H + c]);
    s2 += __half2float(dY[(r + 2) * H + c]); s3 += __half2float(dY[(r + 3) * H + c]);
  }
  for (; r < r1; ++r) s0 += __half2float(dY[r * H + c]);
  atomicAdd(gb + c, ((s0 + s1) + (s2 + s3)) * INV_LS);
}

// ---------------------------------------------------------------------------------------------
// PE backward: d/d(proj_d) = pi sum_k 2^k g[k,d] cos(pi 2^k proj_d);  dB[d][i] += dproj_d * t_i
// ---------------------------------------------------------------------------------------------
// d(loss)/d(proj_d) x 2^8 / pi from a dE row g: sum_k 2^k g[k,d] cos(pi 2^k proj_d), the cosines of sincos_ladder6
__device__ __forceinline__ float pe_dproj(const float* g, int d, const float (&c)[6]) {
  float dp = g[3 + d] * c[0];
  dp = fmaf(2.f * g[3 + VMB_NDIRS + d], c[1], dp);
  dp = fmaf(4.f * g[3 + 2 * VMB_NDIRS + d], c[2], dp);
  dp = fmaf(8.f * g[3 + 3 * VMB_NDIRS + d], c[3], dp);
  dp = fmaf(16.f * g[E1W + d], c[4], dp);
  return fmaf(32.f * g[E1W + VMB_NDIRS + d], c[5], dp);
}
constexpr int PEB_LD = 145;      // odd row stride (floats): per-thread row reads are bank-conflict free
constexpr int PEB_SMEM = 128 * PEB_LD * 4;
// the dE rows of points [p0, p0 + 128) into shared memory [128][PEB_LD]: they are one contiguous 128 x 576 B span,
// read as flat float4 loads, 12 in flight per thread
__device__ __forceinline__ void stage_de_rows(float* sg, const float* __restrict__ dE, long long p0, long long P) {
  const long long rows = min(128LL, P - p0);
  const int n4 = (int)rows * (EW / 4);
  const float4* src = reinterpret_cast<const float4*>(dE + p0 * EW);
#pragma unroll 1
  for (int base = 0; base < n4; base += 12 * 128) {
    float4 q[12];
#pragma unroll
    for (int u = 0; u < 12; ++u) {
      const int i = base + u * 128 + threadIdx.x;
      q[u] = i < n4 ? src[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 12; ++u) {
      const int i = base + u * 128 + threadIdx.x;
      if (i < n4) {
        const int r = i / (EW / 4), c = (i - r * (EW / 4)) * 4;
        float* d = sg + r * PEB_LD + c;
        d[0] = q[u].x; d[1] = q[u].y; d[2] = q[u].z; d[3] = q[u].w;
      }
    }
  }
}
__global__ void __launch_bounds__(128) k_lw_pe_bwd(const float* __restrict__ pcs, const float* __restrict__ dirs,
                                                   const float* __restrict__ scale_ptr, long long P,
                                                   const float* __restrict__ dE, float* __restrict__ gB) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  extern __shared__ float sg[];                 // [128 points][PEB_LD]: the dE rows of this block, staged coalesced
  const float scale = *scale_ptr;
  __shared__ float st[3][129];
  const long long p0 = (long long)blockIdx.x * 128;
  const long long p = p0 + threadIdx.x;
  stage_de_rows(sg, dE, p0, P);
  float t0 = 0.f, t1 = 0.f, t2 = 0.f;
  const bool ok = p < P;
  if (ok) { t0 = pcs[p * 3] / scale; t1 = pcs[p * 3 + 1] / scale; t2 = pcs[p * 3 + 2] / scale; }
  st[0][threadIdx.x] = t0; st[1][threadIdx.x] = t1; st[2][threadIdx.x] = t2;
  __syncthreads();
  const float* g = sg + threadIdx.x * PEB_LD;
  float dpv[VMB_NDIRS];
#pragma unroll
  for (int d = 0; d < VMB_NDIRS; ++d) {
    float dp = 0.f;
    if (ok) {
      float s[6], c[6];
      sincos_ladder6(fmaf(__ldg(dirs + d * 3 + 2), t2, fmaf(__ldg(dirs + d * 3 + 1), t1, __ldg(dirs + d * 3) * t0)), s, c);
      dp = pe_dproj(g, d, c) * (VMB_PI_F * INV_LS);
    }
    dpv[d] = dp;
  }
  __syncthreads();                               // everyone is done reading its dE row: reuse sg as [21][129]
#pragma unroll
  for (int d = 0; d < VMB_NDIRS; ++d) sg[d * 129 + threadIdx.x] = dpv[d];
  __syncthreads();
  if (threadIdx.x < VMB_NDIRS * 3) {
    const int d = threadIdx.x / 3, i = threadIdx.x - d * 3;
    float s = 0.f;
    for (int q = 0; q < 128; ++q) s = fmaf(sg[d * 129 + q], st[i][q], s);
    atomicAdd(gB + threadIdx.x, s);
  }
}

// ---------------------------------------------------------------------------------------------
// host orchestration: one object at a time (wide ensembles have one or very few objects)
// ---------------------------------------------------------------------------------------------
// (k_track_lw.cuh uses it too, and undefines it)
#define LW_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { err = std::string(#expr) + ": " + cudaGetErrorString(e_); return VMB_E_CUDA; } } while (0)

// f(std::integral_constant<int, H>) for the layer-wise widths, once the driver's tensor-map encoder is there; `what`
// names the path in the error
template <class F>
static int for_hidden(int H, const char* what, std::string& err, F&& f) {
  if (!get_encode()) { err = "cuTensorMapEncodeTiled not available from the driver"; return VMB_E_CUDA; }
  switch (H) {
    case 64:  return f(std::integral_constant<int, 64>());
    case 128: return f(std::integral_constant<int, 128>());
    case 256: return f(std::integral_constant<int, 256>());
  }
  err = std::string(what) + ": hidden must be 64, 128 or 256";
  return VMB_E_UNSUPPORTED;
}

// programmatic dependent launch pays where the step is a chain of short single-wave kernels (background model, iMAP
// shards: -3..5 %); at the full iMAP shape the kernels are HBM-bound for tens of microseconds and the early launch of
// the successor only takes resources from them (+1 %): armed below 64 K points only
static bool pdl_ok(long long np) { return np <= 65536; }

// blocks of a heads / render launch over R rays: four rays each, no more than stay resident with their row buffers
template <int H>
static int hr_blocks(int R, int n_sm) {
  const int hr_per_sm = std::max(1, std::min(8, (int)(227 * 1024 / (hr_smem<H>() + 6 * 1024))));
  return std::min((R + 3) / 4, n_sm * hr_per_sm);
}

// ---------------------------------------------------------------------------------------------
// GEMM launches of one object, shared by the training step (step_object) and the tracking path (k_track_lw.cuh)
// ---------------------------------------------------------------------------------------------
// forward: the five layers E -> X1 -> X2 -> X3 -> X4 -> XC (model.py:54-85); Pb = the object's fp32 param row (biases),
// Wi = its fp16 image.  Each launch follows its predecessor directly on `st` (k_lw_pe first): armed when pdl_ok.
template <int H>
static cudaError_t forward_gemms(Workspace& ws, const VmbLayout& L, const float* Pb, const __half* Wi, long long np, cudaStream_t st) {
  const int mt = (int)((np + BM - 1) / BM);
  const Operand none{nullptr, 0, 0, 0};
  auto opX = [&](const __half* x) { return Operand{x, np, H, H}; };
  const Operand opE1{ws.E, np, E1W, EW}, opE2{ws.E + E1W, np, E2W, EW};
  auto fwd = [&](const Operand& a1, const Operand& a2, int K1, int K2, long long woff, int ldw, int boff, __half* out) {
    GemmArgs g; memset(&g, 0, sizeof(g));
    g.M = (int)np; g.N = H; g.K1 = K1; g.K2 = K2; g.bias = Pb + boff; g.out16 = out; g.ldo = H; g.scale = 1.0f;
    if (pdl_ok(np)) pdl_arm();                      // follows k_lw_pe / the previous layer directly on `st`
    return launch_gemm_auto<0, EPI_RELU_F16>(a1, a2, Operand{Wi + woff, H, ldw, ldw}, g, mt, (H + BN - 1) / BN, st);
  };
  cudaError_t e = fwd(opE1, none, E1W, 0, 0, 96, L.o_bin, ws.X1);
  if (e == cudaSuccess) e = fwd(opX(ws.X1), none, H, 0, off_m1(H), H, L.o_bm1, ws.X2);
  if (e == cudaSuccess) e = fwd(opX(ws.X2), opE1, H, E1W, off_cat(H), H + 96, L.o_bcat, ws.X3);
  if (e == cudaSuccess) e = fwd(opX(ws.X3), none, H, 0, off_m2(H), H, L.o_bm2, ws.X4);
  if (e == cudaSuccess) e = fwd(opX(ws.X4), opE2, H, E2W, off_cl(H), H + 48, L.o_bcl, ws.XC);
  return e;
}

// The input-gradient chain from dYc (and dalpha_s) to the embedding gradient dE, one GEMM per member, in this order:
// de_colour (the colour block of dE), dy4 (with the rank-1 d_alpha w_a term) -> dYa, dy3 -> dYb, dy2 -> dYa, dy1 -> dYc, demb1
// (the emb1 block of dE from dY3 and dY1).  Wi = the object's fp16 image, w_a its fp32 out_alpha row.  Each member
// launches on `st`; the caller arms it, or puts its own work in between.
template <int H>
struct InputGrads {
  Workspace& ws;
  const __half* Wi;
  const float* w_a;
  long long np;
  cudaStream_t st;

  // out = gate(x_prev) * (dY @ W[:, woff block] (+ rank-1 r1row x r1col))
  cudaError_t gate(const __half* dY, long long woff, int ldw, const __half* xprev, __half* out, const float* r1row = nullptr,
                   const float* r1col = nullptr) const {
    GemmArgs g; memset(&g, 0, sizeof(g));
    g.M = (int)np; g.N = H; g.K1 = H; g.out16 = out; g.ldo = H; g.gate = xprev; g.ldg = H; g.r1_row = r1row; g.r1_col = r1col;
    g.r1_stride = 1; g.scale = 1.0f;
    const Operand none{nullptr, 0, 0, 0};
    return launch_gemm_auto<1, EPI_GATE_F16>(Operand{dY, np, H, H}, none, Operand{Wi + woff, H, H, ldw}, g,
                                             (int)((np + BM - 1) / BM), (H + BN - 1) / BN, st);
  }
  // dE[:, ecol:ecol+N] (=|+=) dY @ W[:, woff block]
  cudaError_t emb(const __half* dY, long long woff, int ldw, int N, int ecol, int accumulate) const {
    GemmArgs g; memset(&g, 0, sizeof(g));
    g.M = (int)np; g.N = N; g.K1 = H; g.out32 = ws.dE + ecol; g.ld32 = EW; g.accumulate = accumulate; g.scale = 1.0f;
    const Operand none{nullptr, 0, 0, 0};
    return launch_gemm_auto<1, EPI_F32>(Operand{dY, np, H, H}, none, Operand{Wi + woff, H, N, ldw}, g, (int)((np + BM - 1) / BM), 1, st);
  }
  cudaError_t de_colour() const { return emb(ws.dYc, off_cl(H) + H, H + 48, E2W, E1W, 0); }
  cudaError_t dy4() const { return gate(ws.dYc, off_cl(H), H + 48, ws.X4, ws.dYa, ws.dalpha_s, w_a); }
  cudaError_t dy3() const { return gate(ws.dYa, off_m2(H), H, ws.X3, ws.dYb); }
  cudaError_t dy2() const { return gate(ws.dYb, off_cat(H), H + 96, ws.X2, ws.dYa); }
  cudaError_t dy1() const { return gate(ws.dYa, off_m1(H), H, ws.X1, ws.dYc); }
  // d emb1 = dY3 @ W_cat[:, H:] + dY1 @ W_in in ONE launch: A = [dY3 | dY1] along K, B = the two weight blocks
  // (two launches, the second accumulating, where the weight-stationary kernel does not fit)
  cudaError_t demb1() const {
    GemmArgs g; memset(&g, 0, sizeof(g));
    g.M = (int)np; g.N = E1W; g.K1 = H; g.K2 = H; g.out32 = ws.dE; g.ld32 = EW; g.accumulate = 0; g.scale = 1.0f;
    const Operand bcat{Wi + off_cat(H) + H, H, E1W, H + 96}, bin{Wi, H, E1W, 96};
    cudaError_t e = launch_gemm_ws<1, EPI_F32>(Operand{ws.dYb, np, H, H}, Operand{ws.dYc, np, H, H}, bcat, g,
                                                (int)((np + BM - 1) / BM), st, &bin);
    if (e == cudaErrorNotSupported) {
      (void)cudaGetLastError();
      e = emb(ws.dYb, off_cat(H) + H, H + 96, E1W, 0, 0);
      if (e == cudaSuccess) e = emb(ws.dYc, 0, 96, E1W, 0, 1);
    }
    return e;
  }
};

template <int H>
static int step_object(Workspace& ws, const VmbLayout& L, const StepParams& sp, const __half* image, int b, cudaStream_t st,
                       std::string& err, long long fwd_p0 = 0, long long fwd_np = 0) {
  // fwd_only (vmb_forward): points [fwd_p0, fwd_p0 + fwd_np) of object b, raw head outputs, no render
  const long long np = sp.fwd_only ? fwd_np : (long long)sp.R * sp.S;
  const float* Pb = sp.params + (size_t)b * L.stride;
  float* G = sp.grads ? sp.grads + (size_t)b * L.stride : nullptr;
  const __half* Wi = image + (size_t)b * img_halves(H);
  const float* pcs = sp.pcs + (size_t)b * sp.pcs_stride + (sp.fwd_only ? fwd_p0 * 3 : 0);
  const float* dirs = Pb + L.o_B;
  const float* scale_p = sp.scale + b;
  const int nblk = (int)((np + 127) / 128);
  const Operand none{nullptr, 0, 0, 0};
  auto arm = [&]() { if (pdl_ok(np)) pdl_arm(); };
  auto opX = [&](const __half* x) { return Operand{x, np, H, H}; };
  const Operand opE1{ws.E, np, E1W, EW}, opE2{ws.E + E1W, np, E2W, EW};

  // ---- forward ----
  LW_TRY(launch_k(k_lw_pe, dim3(nblk), dim3(128), 0, st, pcs, dirs, scale_p, np, ws.E));
  LW_TRY(forward_gemms<H>(ws, L, Pb, Wi, np, st));
  if (sp.fwd_only) {
    arm();
    LW_TRY(launch_k(k_lw_heads<H>, dim3(nblk), dim3(128), 0, st, (const __half*)ws.X4, (const __half*)ws.XC, Pb, L, np,
                    sp.out_alpha + (size_t)b * sp.alpha_stride + fwd_p0, sp.out_colour + (size_t)b * sp.colour_stride + fwd_p0 * 3, 1));
    return 0;
  }
  RenderArgs ra;
  ra.b = b; ra.R = sp.R; ra.S = sp.S; ra.B = sp.B;
  ra.z = sp.z + (size_t)b * sp.z_stride; ra.gt_depth = sp.gt_depth + (size_t)b * sp.gt_depth_stride;
  ra.gt_colour = sp.gt_colour + (size_t)b * sp.gt_colour_stride; ra.sem = sp.sem + (size_t)b * sp.sem_stride;
  ra.mask = sp.mask + (size_t)b * sp.mask_stride; ra.counts = sp.counts; ra.cs = sp.cs; ra.os = sp.os; ra.backward = sp.backward;
  ra.loss_terms = sp.loss_terms; ra.r_depth = sp.r_depth; ra.r_var = sp.r_var; ra.r_colour = sp.r_colour; ra.r_opacity = sp.r_opacity;
  // heads + render + loss (+ head gradients when training) in one launch
  int dev = 0;
  cudaGetDevice(&dev);
  const int n_sm = sm_count(dev);
  LW_TRY(smem_limit_once<k_lw_heads_render<H>>(dev, hr_smem<H>()));
  arm();
  LW_TRY(launch_k(k_lw_heads_render<H>, dim3(hr_blocks<H>(sp.R, n_sm)), dim3(128), (size_t)hr_smem<H>(), st, ra,
                  (const __half*)ws.X4, (const __half*)ws.XC, Pb, L, ws.dYc, ws.dh16, ws.dalpha_s, G));
  if (!sp.backward) return 0;

  // ---- backward ----
  // split over points: enough z slices that the widest weight-gradient GEMM (2 x 2 output tiles) fills the machine
  // (one resident CTA per SM) at any point count, bounded below so a slice still amortises its pipeline fill
  const int ksplit = (int)std::min<long long>(4096, std::max<long long>(512, ((np * 4 / n_sm + BK - 1) / BK) * BK));
  const int zs = (int)((np + ksplit - 1) / ksplit);
  const int cs_rows = (int)std::max<long long>(64, (np + 4 * n_sm - 1) / (4 * n_sm));       // bias column sums: ~4 blocks per SM
  // weight gradient: G[o*ldm + n] += sum_p dY[p][o] * X[p][n]   (A = dY^T, B = X, both MN-major, split over points)
  LW_TRY(ws.ensure_streams());
  cudaStream_t sd = ws.side;
  auto fork = [&](int i) { cudaEventRecord(ws.ev_main[i], st); return cudaStreamWaitEvent(sd, ws.ev_main[i], 0); };
  auto wgrad = [&](const __half* dY, const Operand& xb, int N, int goff, int ldm, int n_valid, int ones_col, int boff) {
    GemmArgs g; memset(&g, 0, sizeof(g));
    g.M = H; g.N = N; g.K1 = (int)np; g.K2 = 0; g.ksplit = ksplit; g.gdst = G + goff; g.ldgd = ldm; g.ldgn = 1; g.n_lo = 0;
    g.n_valid = n_valid; g.ones_col = ones_col; g.gbias = boff >= 0 ? G + boff : nullptr; g.scale = INV_LS;
    return launch_gemm<1, 1, EPI_ATOMIC>(Operand{dY, np, H, H}, none, xb, g, (H + BM - 1) / BM, (N + BN - 1) / BN, zs, sd);
  };
  const InputGrads<H> ig{ws, Wi, Pb + L.o_Wa, np, st};
  // heads: dW_a[o] = sum_p d_a fc4[p][o]; dW_oc[c][o] = sum_p d_rc[c] hc[p][o]   (B = dh16 [P][8], columns 0 / 1..3)
  {
    GemmArgs g; memset(&g, 0, sizeof(g));
    g.M = H; g.N = 8; g.K1 = (int)np; g.ksplit = ksplit; g.ldgd = 1; g.scale = INV_LS; g.ones_col = -1;
    g.gdst = G + L.o_Wa; g.ldgn = 0; g.n_lo = 0; g.n_valid = 1;
    LW_TRY(fork(0));                                    // dYc (= d colour hidden), dh16 ready: heads + color_linear wgrads on the side stream
    LW_TRY((launch_gemm<1, 1, EPI_ATOMIC>(Operand{ws.X4, np, H, H}, none, Operand{ws.dh16, np, 8, 8}, g, (H + BM - 1) / BM, 1, zs, sd)));
    g.gdst = G + L.o_Woc - H; g.ldgn = H; g.n_lo = 1; g.n_valid = 4;
    arm();
    LW_TRY((launch_gemm<1, 1, EPI_ATOMIC>(Operand{ws.XC, np, H, H}, none, Operand{ws.dh16, np, 8, 8}, g, (H + BM - 1) / BM, 1, zs, sd)));
  }
  // color_linear
  arm();
  LW_TRY(wgrad(ws.dYc, opX(ws.X4), H, L.o_Wcl, H + L.e2, H, -1, -1));
  arm();
  LW_TRY(wgrad(ws.dYc, opE2, E2W, L.o_Wcl + H, H + L.e2, L.e2, ONES2, L.o_bcl));
  LW_TRY(ig.de_colour());                                     // first kernel on `st` after the fork: not armed
  arm();
  LW_TRY(ig.dy4());
  // mid2
  LW_TRY(fork(1));
  LW_TRY(wgrad(ws.dYa, opX(ws.X3), H, L.o_Wm2, H, H, -1, -1));
  arm();                                          // follows this layer's weight-gradient GEMM directly on the side stream
  LW_TRY(launch_k(k_lw_colsum, dim3((unsigned)((np + cs_rows - 1) / cs_rows)), dim3(256), 0, sd, (const __half*)ws.dYa, np, H, cs_rows, G + L.o_bm2));
  LW_TRY(cudaEventRecord(ws.ev_side[0], sd));           // the side stream is done reading dYc (dY of color_linear) and dYa (dY4)
  LW_TRY(ig.dy3());
  // cat_layer
  LW_TRY(fork(2));
  LW_TRY(wgrad(ws.dYb, opX(ws.X2), H, L.o_Wcat, H + VMB_E1, H, -1, -1));
  arm();
  LW_TRY(wgrad(ws.dYb, opE1, E1W, L.o_Wcat + H, H + VMB_E1, VMB_E1, ONES1, L.o_bcat));
  LW_TRY(cudaStreamWaitEvent(st, ws.ev_side[0], 0));    // dYa / dYc are about to be overwritten
  LW_TRY(ig.dy2());                                     // dY3 stays in dYb
  // mid1
  LW_TRY(fork(3));
  LW_TRY(wgrad(ws.dYa, opX(ws.X1), H, L.o_Wm1, H, H, -1, -1));
  arm();                                          // follows this layer's weight-gradient GEMM directly on the side stream
  LW_TRY(launch_k(k_lw_colsum, dim3((unsigned)((np + cs_rows - 1) / cs_rows)), dim3(256), 0, sd, (const __half*)ws.dYa, np, H, cs_rows, G + L.o_bm1));
  LW_TRY(ig.dy1());                                     // dYc is free since color_linear
  // in_layer
  LW_TRY(fork(4));
  LW_TRY(wgrad(ws.dYc, opE1, E1W, L.o_Win, VMB_E1, VMB_E1, ONES1, L.o_bin));
  LW_TRY(cudaEventRecord(ws.ev_side[1], sd));
  LW_TRY(ig.demb1());
  LW_TRY(smem_limit_once<k_lw_pe_bwd>(dev, PEB_SMEM));
  arm();                                         // follows the embedding-gradient GEMM directly on `st`
  LW_TRY(launch_k(k_lw_pe_bwd, dim3(nblk), dim3(128), (size_t)PEB_SMEM, st, pcs, dirs, scale_p, np, (const float*)ws.dE, G + L.o_B));
  LW_TRY(cudaStreamWaitEvent(st, ws.ev_side[1], 0));    // join: every weight-gradient GEMM of this object has been enqueued before what follows
  LW_TRY(cudaGetLastError());
  return 0;
}

// forward only (vmb_forward): chunks of FWD_CHUNK points so the activation workspace stays bounded for 256^3 grids
constexpr long long FWD_CHUNK = 1LL << 18;
static int launch_forward(Workspace& ws, const VmbLayout& L, const StepParams& sp, const void* image, cudaStream_t st, std::string& err) {
  return for_hidden(L.H, "layer-wise path", err, [&](auto h) -> int {
    const long long N = sp.R;
    LW_TRY(ws.grow(std::min(N, FWD_CHUNK), L.H, stream_capturing(st)));
    for (int b = 0; b < sp.B; ++b)
      for (long long p0 = 0; p0 < N; p0 += FWD_CHUNK)
        if (const int rc = step_object<decltype(h)::value>(ws, L, sp, (const __half*)image, b, st, err, p0, std::min(FWD_CHUNK, N - p0)))
          return rc;
    return 0;
  });
}

static int launch_step(Workspace& ws, const VmbLayout& L, const StepParams& sp, const void* image, cudaStream_t st, std::string& err) {
  return for_hidden(L.H, "layer-wise path", err, [&](auto h) -> int {
    if (sp.S > 32) { err = "layer-wise path: n_samples > 32"; return VMB_E_UNSUPPORTED; }
    LW_TRY(ws.grow((long long)sp.R * sp.S, L.H, stream_capturing(st)));
    for (int b = 0; b < sp.B; ++b)
      if (const int rc = step_object<decltype(h)::value>(ws, L, sp, (const __half*)image, b, st, err)) return rc;
    return 0;
  });
}

}  // namespace lw
