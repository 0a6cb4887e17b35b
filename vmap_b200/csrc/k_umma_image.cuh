// Weight image and shared device helpers of the hidden-32 tensor-core step kernel (k_step_fused.cuh).
//
// Weight image (per object, um::IMG_BYTES, written by the AdamW finisher / k_adamw / k_build_image, staged into shared
// memory with ONE bulk async copy per (CTA, object)): the 14 OccupancyMap tensors rounded to fp16 and pre-arranged in
// the tensor core's shared-memory operand layout -- SWIZZLE_NONE 8x8 core matrices, W[o][k] at
// (k/8)*512 + o*16 + (k%8)*2 -- which serves as a K-major B operand (forward) and as an MN-major B operand (dgrad);
// columns permuted to the kernel's embedding order, a zero column under each constant-1 feature; then fp32 biases and
// the PE directions stored component-major ([x|y|z][24]) so four directions' components arrive with one 16-byte load.
//
// Feature order inside the embedding blocks is chosen for the PE recurrence (one sincos per direction, then angle
// doubling), and each block carries a constant-1 column so the bias gradients fall out of the wgrad MMAs.
// dY operands carry a static loss scale of 2^8.
#pragma once
#include "common.cuh"
#include "umma_ptx.cuh"

namespace um {

// weight image (bytes)
constexpr int IMG_WIN = 0, IMG_WM1 = 6144, IMG_WCAT = 8192, IMG_WM2 = 16384, IMG_WCL = 18432;
constexpr int IMG_WA16 = 23552, IMG_WOC16 = 24576, IMG_F32 = 25600;
// fp32 section (float index relative to IMG_F32); directions: F_DIRS + c * DIRS_PITCH + d
constexpr int F_BIN = 0, F_BM1 = 32, F_BCAT = 64, F_BM2 = 96, F_BCL = 128, F_BA = 160, F_BOC = 161, F_DIRS = 168, DIRS_PITCH = 24;
constexpr int IMG_BYTES = 26624;
constexpr float LS = 256.0f, INV_LS = 1.0f / 256.0f;

// ---- column maps ------------------------------------------------------------------------
// emb1 block (96 cols): 0 = const 1, 1..3 = xyz/scale, 4..7 = dir 20 (k=0..3),
// 8i+e (i=1..10) = dir 2(i-1)+e/4, k=e%4; 88..95 = 0.
__host__ __device__ inline int emb1_col_to_j(int c) {     // -> reference emb index, -2 ones, -1 pad
  if (c == 0) return -2;
  if (c < 4) return c - 1;
  if (c < 8) return 3 + (c - 4) * VMB_NDIRS + 20;
  if (c >= 88) return -1;
  const int i = c >> 3, e = c & 7;
  return 3 + (e & 3) * VMB_NDIRS + 2 * (i - 1) + (e >> 2);
}
__host__ __device__ inline int j_to_emb1_col(int j) {
  if (j < 3) return 1 + j;
  const int k = (j - 3) / VMB_NDIRS, d = (j - 3) % VMB_NDIRS;
  if (d == 20) return 4 + k;
  return 8 * (d / 2 + 1) + (d & 1) * 4 + k;
}
// emb2 block (48 cols): 8i+e (i=0..4) = dir 4i+e/2, k=4+e%2; 40,41 = dir 20 (k=4,5); 42 = const 1.
__host__ __device__ inline int emb2_col_to_j2(int c) {    // -> index into the reference's emb[87:], -2 ones, -1 pad
  if (c == 42) return -2;
  if (c > 42) return -1;
  int d, k;
  if (c >= 40) { d = 20; k = 4 + (c - 40); } else { d = 4 * (c >> 3) + ((c & 7) >> 1); k = 4 + (c & 1); }
  return 3 + k * VMB_NDIRS + d - VMB_E1;
}
__host__ __device__ inline int j2_to_emb2_col(int j2) {
  const int j = j2 + VMB_E1;
  const int k = (j - 3) / VMB_NDIRS, d = (j - 3) % VMB_NDIRS;
  if (d == 20) return 40 + (k - 4);
  return 8 * (d / 4) + (d & 3) * 2 + (k - 4);
}
// half index of W[o][c] in a 32-row matrix / of W[j][o] in a 16-row (heads) matrix
__host__ __device__ inline int widx32(int base_bytes, int o, int c) { return (base_bytes + (c >> 3) * 512 + o * 16 + (c & 7) * 2) >> 1; }
__host__ __device__ inline int widx16(int base_bytes, int j, int o) { return (base_bytes + (o >> 3) * 256 + j * 16 + (o & 7) * 2) >> 1; }

__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// sigmoid on the fast path: MUFU.EX2 + MUFU.RCP (rel. error ~1e-6, far below the fp16 operand noise)
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ uint32_t relu_h2(uint32_t x) {
  __half2 h = __hmax2(*reinterpret_cast<__half2*>(&x), __float2half2_rn(0.f));
  return *reinterpret_cast<uint32_t*>(&h);
}
// dy * (h > 0), packed
__device__ __forceinline__ uint32_t gate_h2(uint32_t dy, uint32_t h) {
  const __half2 m = __hgt2(*reinterpret_cast<__half2*>(&h), __float2half2_rn(0.f));
  __half2 r = __hmul2(*reinterpret_cast<__half2*>(&dy), m);
  return *reinterpret_cast<uint32_t*>(&r);
}
// Bring-up safety net: a protocol bug traps (CUDA error) instead of hanging the GPU.
#ifndef VMB_SPIN_LIMIT
#define VMB_SPIN_LIMIT 50000000u
#endif
__device__ __forceinline__ void mbar_wait_or_trap(uint64_t* bar, uint32_t parity) {
#pragma unroll 1
  for (uint32_t i = 0; i < VMB_SPIN_LIMIT; ++i)
    if (ptx::mbar_try_wait(bar, parity)) return;
  __trap();
}
// sin(pi 2^k x), k = 0..5: one MUFU sin/cos pair, then angle doubling
__device__ __forceinline__ void sin_ladder(float proj, float (&s)[6]) {
  const float r = proj - 2.0f * rintf(0.5f * proj);          // exact: sin(pi x) has period 2
  s[0] = __sinf(VMB_PI_F * r);
  float c = __cosf(VMB_PI_F * r);
#pragma unroll
  for (int k = 1; k < 6; ++k) {
    const float s2 = s[k - 1] + s[k - 1];
    s[k] = s2 * c;
    c = fmaf(-s2, s[k - 1], 1.0f);
  }
}
// four independent sin ladders interleaved (ILP 4)
__device__ __forceinline__ void sin_ladder4(const float (&proj)[4], float (&s)[4][6]) {
  float c[4];
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const float r = proj[d] - 2.0f * rintf(0.5f * proj[d]);
    s[d][0] = __sinf(VMB_PI_F * r);
    c[d] = __cosf(VMB_PI_F * r);
  }
#pragma unroll
  for (int k = 1; k < 6; ++k)
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const float s2 = s[d][k - 1] + s[d][k - 1];
      s[d][k] = s2 * c[d];
      c[d] = fmaf(-s2, s[d][k - 1], 1.0f);
    }
}
__device__ __forceinline__ void cos_ladder4(const float (&proj)[4], float (&c)[4][6]) {
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const float r = proj[d] - 2.0f * rintf(0.5f * proj[d]);
    c[d][0] = __cosf(VMB_PI_F * r);
  }
#pragma unroll
  for (int k = 1; k < 6; ++k)
#pragma unroll
    for (int d = 0; d < 4; ++d) c[d][k] = fmaf(c[d][k - 1] + c[d][k - 1], c[d][k - 1], -1.0f);
}
// cos(pi 2^k x), k = 0..5
__device__ __forceinline__ void cos_ladder(float proj, float (&c)[6]) {
  const float r = proj - 2.0f * rintf(0.5f * proj);
  c[0] = __cosf(VMB_PI_F * r);
#pragma unroll
  for (int k = 1; k < 6; ++k) c[k] = fmaf(c[k - 1] + c[k - 1], c[k - 1], -1.0f);
}


// ---- fp32 pairs: two directions per value (plain fp32 arithmetic on each half) -------------------------------------
__device__ __forceinline__ uint64_t pk2(float lo, float hi) { uint64_t r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void upk2(uint64_t v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1); upk2(b, b0, b1); upk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}

// Front half of the ladders: range reduction (sin/cos(pi x) have period 2) and the MUFU sin / cos of four directions
// held as two packed pairs (d0,d1 | d2,d3).  Split from the doubling recurrence so that the caller can issue the next
// four directions' front (shared-memory loads, FRND, MUFU: the long latencies) before the current four's recurrence.
__device__ __forceinline__ void sincos4_x2(uint64_t pj01, uint64_t pj23, uint64_t& s01, uint64_t& s23, uint64_t& c01, uint64_t& c23) {
  float p[4], s[4], c[4];
  upk2(pj01, p[0], p[1]); upk2(pj23, p[2], p[3]);
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const float r = p[d] - 2.0f * rintf(0.5f * p[d]);
    s[d] = __sinf(VMB_PI_F * r);
    c[d] = __cosf(VMB_PI_F * r);
  }
  s01 = pk2(s[0], s[1]); s23 = pk2(s[2], s[3]); c01 = pk2(c[0], c[1]); c23 = pk2(c[2], c[3]);
}
__device__ __forceinline__ void cos4_x2(uint64_t pj01, uint64_t pj23, uint64_t& c01, uint64_t& c23) {
  float p[4], c[4];
  upk2(pj01, p[0], p[1]); upk2(pj23, p[2], p[3]);
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const float r = p[d] - 2.0f * rintf(0.5f * p[d]);
    c[d] = __cosf(VMB_PI_F * r);
  }
  c01 = pk2(c[0], c[1]); c23 = pk2(c[2], c[3]);
}
// sin(pi 2^k x), k = 0..5: angle doubling on pairs, same recurrence as sin_ladder4
__device__ __forceinline__ void sin_doubling4_x2(uint64_t s01, uint64_t s23, uint64_t c01, uint64_t c23, float (&s)[4][6]) {
  const uint64_t one = pk2(1.0f, 1.0f), neg = pk2(-1.0f, -1.0f);
  upk2(s01, s[0][0], s[1][0]); upk2(s23, s[2][0], s[3][0]);
#pragma unroll
  for (int k = 1; k < 6; ++k) {
    const uint64_t d01 = add2(s01, s01), d23 = add2(s23, s23);
    const uint64_t n01 = mul2(d01, c01), n23 = mul2(d23, c23);
    c01 = fma2(mul2(d01, s01), neg, one); c23 = fma2(mul2(d23, s23), neg, one);
    s01 = n01; s23 = n23;
    upk2(s01, s[0][k], s[1][k]); upk2(s23, s[2][k], s[3][k]);
  }
}
// cos(pi 2^k x), k = 0..5, four directions as two packed pairs
__device__ __forceinline__ void cos_doubling4_x2(uint64_t c01, uint64_t c23, float (&c)[4][6]) {
  const uint64_t neg = pk2(-1.0f, -1.0f);
  upk2(c01, c[0][0], c[1][0]); upk2(c23, c[2][0], c[3][0]);
#pragma unroll
  for (int k = 1; k < 6; ++k) {
    c01 = fma2(add2(c01, c01), c01, neg); c23 = fma2(add2(c23, c23), c23, neg);
    upk2(c01, c[0][k], c[1][k]); upk2(c23, c[2][k], c[3][k]);
  }
}
// projections of a point on directions 4q .. 4q+3 (component-major direction table: one 16-byte load per component)
__device__ __forceinline__ void project4(const float* Bd, int q, uint64_t t0, uint64_t t1, uint64_t t2, uint64_t& pj01, uint64_t& pj23) {
  const ulonglong2 bx = *reinterpret_cast<const ulonglong2*>(Bd + 4 * q);
  const ulonglong2 by = *reinterpret_cast<const ulonglong2*>(Bd + DIRS_PITCH + 4 * q);
  const ulonglong2 bz = *reinterpret_cast<const ulonglong2*>(Bd + 2 * DIRS_PITCH + 4 * q);
  pj01 = fma2(bz.x, t2, fma2(by.x, t1, mul2(bx.x, t0)));
  pj23 = fma2(bz.y, t2, fma2(by.y, t1, mul2(bx.y, t0)));
}

}  // namespace um

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
static int umma_image_bytes() { return um::IMG_BYTES; }

// param index -> location in the image: t >= 0 half index; t <= -2 float word index -(t+2); -1 none
static void umma_fill_image_index(const VmbLayout& L, int* idx) {
  using namespace um;
  for (int i = 0; i < L.P; ++i) idx[i] = -1;
  auto fslot = [](int f) { return -(IMG_F32 / 4 + f) - 2; };
  const int H = 32;
  for (int o = 0; o < H; ++o) {
    for (int j = 0; j < VMB_E1; ++j) idx[L.o_Win + o * VMB_E1 + j] = widx32(IMG_WIN, o, j_to_emb1_col(j));
    idx[L.o_bin + o] = fslot(F_BIN + o);
    for (int k = 0; k < H; ++k) idx[L.o_Wm1 + o * H + k] = widx32(IMG_WM1, o, k);
    idx[L.o_bm1 + o] = fslot(F_BM1 + o);
    for (int k = 0; k < H + VMB_E1; ++k)
      idx[L.o_Wcat + o * (H + VMB_E1) + k] = widx32(IMG_WCAT, o, k < H ? k : H + j_to_emb1_col(k - H));
    idx[L.o_bcat + o] = fslot(F_BCAT + o);
    for (int k = 0; k < H; ++k) idx[L.o_Wm2 + o * H + k] = widx32(IMG_WM2, o, k);
    idx[L.o_bm2 + o] = fslot(F_BM2 + o);
    for (int k = 0; k < H + L.e2; ++k)
      idx[L.o_Wcl + o * (H + L.e2) + k] = widx32(IMG_WCL, o, k < H ? k : H + j2_to_emb2_col(k - H));
    idx[L.o_bcl + o] = fslot(F_BCL + o);
    idx[L.o_Wa + o] = widx16(IMG_WA16, 0, o);
    for (int c = 0; c < 3; ++c) idx[L.o_Woc + c * H + o] = widx16(IMG_WOC16, 1 + c, o);
  }
  idx[L.o_ba] = fslot(F_BA);
  for (int c = 0; c < 3; ++c) idx[L.o_boc + c] = fslot(F_BOC + c);
  for (int d = 0; d < VMB_NDIRS; ++d)
    for (int c = 0; c < 3; ++c) idx[L.o_B + d * 3 + c] = fslot(F_DIRS + c * DIRS_PITCH + d);      // component-major
}

