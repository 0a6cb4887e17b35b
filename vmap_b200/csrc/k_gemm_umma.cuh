// wgmma GEMMs of the layer-wise path for wide models (hidden 64 / 128 / 256: background model, iMAP whole-scene
// model), where one object's weights and a tile's activations no longer fit in shared memory together and the layers
// run as separate launches over all points.
//
//   D[M][N] (+)= A[M][K] * B[N][K]^T        fp16 operands from shared memory, fp32 accumulate in registers
//
// Two kernels share the operand conventions below:
//   k_gemm_umma  generic persistent kernel: 128 x 128 output tiles, K in chunks of 64, 4-stage TMA -> mbarrier ring,
//                warp 8 = TMA producer (one elected lane), warps 0..7 = two consumer warpgroups.  Warpgroup g owns the
//                tile's columns 64g .. 64g+63: two wgmma.m64n64k16 per K step (rows 0..63 and 64..127), then the
//                epilogue on its own accumulators.  Used for wgrad (split-K over points, atomics) and for the forward
//                layers whose weights exceed the weight-stationary budget.
//   k_gemm_ws    weight-stationary kernel for the skinny forward / dgrad GEMMs (see its header further down).
// * Operand stages use the 128-byte-swizzle canonical layouts, written by TMA (CU_TENSOR_MAP_SWIZZLE_128B, 128-byte
//   inner box so the TMA engine moves full lines):
//     K-major  operand, global [rows][ld]  (K contiguous):  2-D box (64 k, 128 rows)  -> [128 rows][128 B]
//        descriptor SWIZZLE_128B, SBO 1024 (8 rows), k-step +32 B inside the swizzle atom, 64 rows = +8192 B
//     MN-major operand, global [K][ld]     (MN contiguous): two 2-D boxes (64 mn, 64 k) -> two [64 k][128 B] panels
//        descriptor SWIZZLE_128B, SBO 1024 (8 k-rows), k-step +2048 B, one panel per 64 rows / columns
//   Out-of-range rows / columns are zero-filled by the TMA engine, so ragged edges need no branches.
// * A may come from two sources concatenated along K (e.g. [fc2 | emb1] for cat_layer).
// * Not pipelined yet: a consumer waits for each K chunk's wgmmas (wait_group 0) before it looks at the next stage, a
//   tile's epilogue does not overlap the next tile's MMAs, and ptxas reports the wgmmas of both kernels as serialised
//   (C7520; the build prints the count).  The TMA ring still runs ahead of the consumers.
// * Epilogues work one output ROW per lane: a warp's accumulator fragments (rows 16w .. 16w+15 of both 64-row halves)
//   are transposed through a per-warp shared-memory tile, 32 columns at a time.
#pragma once
#include "common.cuh"
#include "umma_ptx.cuh"
#include <cuda.h>
#include <algorithm>

namespace lw {

constexpr int BM = 128, BN = 128, BK = 64, NSTAGE = 4;
constexpr int STAGE_BYTES = (BM + BN) * BK * 2;             // 32 KB
constexpr int N_CWARPS = 8;                                 // consumer warps (two warpgroups)
constexpr int EPI_SCRATCH = 32 * 144;                       // per consumer warp: fragment transposition tile, then the epilogue's staging tile
constexpr int GEMM_SMEM = NSTAGE * STAGE_BYTES + 1024 + N_CWARPS * EPI_SCRATCH;      // + barriers
constexpr int GEMM_THREADS = 32 * (N_CWARPS + 1);
constexpr float LS = 256.0f, INV_LS = 1.0f / 256.0f;

enum Epi { EPI_RELU_F16 = 0, EPI_GATE_F16 = 1, EPI_F32 = 2, EPI_ATOMIC = 3 };

// Host side of programmatic dependent launch.  The orchestrator arms `t_pdl_next` right before a launch that directly
// follows another kernel of the chain on the same stream; `launch_k` consumes it.  Every kernel of the layer-wise path
// executes `ptx::pdl_wait()` before it touches anything its predecessor wrote, so an armed launch only overlaps its
// prologue (and the launch latency itself) with the predecessor's tail.
static thread_local bool t_pdl_next = false;
static inline void pdl_arm() { t_pdl_next = true; }
template <typename... KArgs, typename... Args>
static cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = t_pdl_next ? 1 : 0;
  t_pdl_next = false;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

struct GemmArgs {
  int M, N;                 // valid output extent
  int K1, K2;               // K taken from A source 1 / source 2 (multiples of 16; K2 may be 0)
  int b_k0;                 // K offset into B for this launch's first chunk (used with split-K on points)
  int b_two;                // weight-stationary kernel: B also comes from two sources (second one covers K >= K1)
  int ksplit;               // K elements per z slice (0 = no split)
  int mt, nt, zt;           // tile counts (filled by launch_gemm)
  // epilogue
  const float* bias;        // [N] (EPI_RELU_F16)
  __half* out16; int ldo;   // fp16 output
  const __half* gate; int ldg;          // EPI_GATE_F16: activation whose sign gates the gradient
  const float* r1_row; const float* r1_col; int r1_stride;   // optional rank-1 term: acc += r1_row[m*r1_stride] * r1_col[n]
  float* out32; int ld32; int accumulate;                    // EPI_F32
  float* gdst; int ldgd; int ldgn; int n_lo; int n_valid; int ones_col; float* gbias;
                            // EPI_ATOMIC: G[m*ldgd + n*ldgn] += acc for n_lo <= n < n_valid; n == ones_col -> gbias[m]
  float scale;              // multiplies the accumulator (loss-scale removal)
};

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(ptx::smem_u32(dst)), "l"(map), "r"(ptx::smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// SWIZZLE_128B shared-memory matrix descriptor
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | ((uint64_t)1 << 62);
}

// Row r (0..31) of a consumer warp's slice of a 128-row tile: rows 16w .. 16w+15 of each 64-row wgmma half
// (m_base = tile row 0 + 16w).
__device__ __forceinline__ int wrow(int m_base, int r) { return m_base + (r & 15) + ((r >> 4) << 6); }

// Accumulator fragments of the two 64-row halves (m64n64: d[4j + 0..1] = row l/4, columns 8j + 2(l%4) + {0, 1};
// d[4j + 2..3] = row + 8) -> v = columns 32 cq .. 32 cq + 31 of warp row `lane` (see wrow), through the warp's tile.
template <int CQ>
__device__ __forceinline__ void frag_rows(const float (&d0)[32], const float (&d1)[32], unsigned char* scratch, int lane, float (&v)[32]) {
  float* t = reinterpret_cast<float*>(scratch);
  const int r = lane >> 2, c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = 4 * (4 * CQ + j);
    t[r * 33 + 8 * j + c] = d0[k];             t[r * 33 + 8 * j + c + 1] = d0[k + 1];
    t[(r + 8) * 33 + 8 * j + c] = d0[k + 2];   t[(r + 8) * 33 + 8 * j + c + 1] = d0[k + 3];
    t[(r + 16) * 33 + 8 * j + c] = d1[k];      t[(r + 16) * 33 + 8 * j + c + 1] = d1[k + 1];
    t[(r + 24) * 33 + 8 * j + c] = d1[k + 2];  t[(r + 24) * 33 + 8 * j + c + 1] = d1[k + 3];
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = t[lane * 33 + j];
  __syncwarp();
}

// Epilogue of one 32-column chunk for the 32 rows of a warp: v = accumulator values of columns nb .. nb+31 of
// row wrow(m_base, lane).  A thread owns one output ROW, so direct stores would touch 32 different
// cache lines per instruction (16 B each); the fp16 / fp32 paths therefore transpose through a per-warp
// shared-memory tile so that each store (and each gate / accumulate load) instruction covers whole 64 B / 128 B
// row segments (8 / 4 rows per instruction).  `stage` = per-warp scratch (EPI_STAGE_F16 / EPI_STAGE_F32 bytes),
// nullptr -> direct per-row access (EPI_ATOMIC, and the generic kernel's EPI_F32).
constexpr int EPI_STAGE_F16 = 32 * 80;      // [32 rows][64 B + 16 B pad]
constexpr int EPI_STAGE_F32 = 32 * 144;     // [32 rows][128 B + 16 B pad]

__device__ __forceinline__ void stage_store_f16(unsigned char* stage, int lane, const uint32_t (&h)[16], __half* out, int ldo,
                                                int m_base, int M, int nb, int N) {
  uint4* mine = reinterpret_cast<uint4*>(stage + lane * 80);
#pragma unroll
  for (int q = 0; q < 4; ++q) mine[q] = make_uint4(h[4 * q], h[4 * q + 1], h[4 * q + 2], h[4 * q + 3]);
  __syncwarp();
  const int piece = lane & 3;
#pragma unroll
  for (int s4 = 0; s4 < 4; ++s4) {
    const int r = 8 * s4 + (lane >> 2), m = wrow(m_base, r);
    const uint4 val = *reinterpret_cast<const uint4*>(stage + r * 80 + piece * 16);
    if (m < M && nb + piece * 8 < N) *reinterpret_cast<uint4*>(out + (size_t)m * ldo + nb + piece * 8) = val;
  }
  __syncwarp();
}

// two fp32 -> packed fp16x2 (lo = first argument), saturating to the largest finite half
__device__ __forceinline__ uint32_t pack_sat(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// `bias` / `r1col` point at 256-entry arrays when they live in shared memory (weight-stationary kernel): they are
// then read as float4 without bounds checks (entries past N are zero).
template <int EPI, bool SMEM_VEC = false>
__device__ __forceinline__ void epi_chunk(const GemmArgs& g, float (&v)[32], int m_base, int lane, int nb, const float* bias,
                                          unsigned char* stage, const uint4* gpre = nullptr, const float* r1col = nullptr) {
  const int m = wrow(m_base, lane);
  if (EPI == EPI_RELU_F16) {
    uint32_t h[16];
    const __half2 zero2 = __float2half2_rn(0.f);
#pragma unroll
    for (int q4 = 0; q4 < 8; ++q4) {
      float4 bv;
      if (SMEM_VEC) bv = *reinterpret_cast<const float4*>(bias + nb + 4 * q4);
      else {
        const int n = min(nb + 4 * q4, g.N - 4);                    // columns past N are never stored
        bv = make_float4(bias[n], bias[n + 1], bias[n + 2], bias[n + 3]);
      }
      uint32_t p0 = pack_sat(fmaf(v[4 * q4], g.scale, bv.x), fmaf(v[4 * q4 + 1], g.scale, bv.y));
      uint32_t p1 = pack_sat(fmaf(v[4 * q4 + 2], g.scale, bv.z), fmaf(v[4 * q4 + 3], g.scale, bv.w));
      __half2 r0 = __hmax2(*reinterpret_cast<__half2*>(&p0), zero2), r1 = __hmax2(*reinterpret_cast<__half2*>(&p1), zero2);
      h[2 * q4] = *reinterpret_cast<uint32_t*>(&r0);
      h[2 * q4 + 1] = *reinterpret_cast<uint32_t*>(&r1);
    }
    stage_store_f16(stage, lane, h, g.out16, g.ldo, m_base, g.M, nb, g.N);
  } else if (EPI == EPI_GATE_F16) {
    const int piece = lane & 3;
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4) {                                // gate rows arrive in the coalesced (8 rows x 64 B) pattern
      const int r = 8 * s4 + (lane >> 2);
      uint4 gv;
      if (gpre) gv = gpre[s4];
      else {
        const int mr = wrow(m_base, r);
        gv = make_uint4(0u, 0u, 0u, 0u);
        if (mr < g.M && nb + piece * 8 < g.N) gv = *reinterpret_cast<const uint4*>(g.gate + (size_t)mr * g.ldg + nb + piece * 8);
      }
      *reinterpret_cast<uint4*>(stage + r * 80 + piece * 16) = gv;
    }
    __syncwarp();
    uint4 gq[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) gq[q] = *reinterpret_cast<const uint4*>(stage + lane * 80 + q * 16);
    __syncwarp();
    const __half2* gh2 = reinterpret_cast<const __half2*>(gq);
    const float r1 = (g.r1_row && m < g.M) ? g.r1_row[(size_t)m * g.r1_stride] : 0.f;
    const __half2 zero2 = __float2half2_rn(0.f);
    uint32_t h[16];
#pragma unroll
    for (int q4 = 0; q4 < 8; ++q4) {
      float a0 = v[4 * q4] * g.scale, a1 = v[4 * q4 + 1] * g.scale, a2 = v[4 * q4 + 2] * g.scale, a3 = v[4 * q4 + 3] * g.scale;
      if (g.r1_row) {
        float4 rc;
        if (SMEM_VEC) rc = *reinterpret_cast<const float4*>(r1col + nb + 4 * q4);
        else {
          const int n = min(nb + 4 * q4, g.N - 4);
          rc = make_float4(g.r1_col[n], g.r1_col[n + 1], g.r1_col[n + 2], g.r1_col[n + 3]);
        }
        a0 = fmaf(r1, rc.x, a0); a1 = fmaf(r1, rc.y, a1); a2 = fmaf(r1, rc.z, a2); a3 = fmaf(r1, rc.w, a3);
      }
      // relu'(x_prev) gate as a 1.0 / 0.0 half2 mask; the saturating pack keeps the product finite
      uint32_t p0 = pack_sat(a0, a1), p1 = pack_sat(a2, a3);
      __half2 r0 = __hmul2(*reinterpret_cast<__half2*>(&p0), __hgt2(gh2[2 * q4], zero2));
      __half2 r1h = __hmul2(*reinterpret_cast<__half2*>(&p1), __hgt2(gh2[2 * q4 + 1], zero2));
      h[2 * q4] = *reinterpret_cast<uint32_t*>(&r0);
      h[2 * q4 + 1] = *reinterpret_cast<uint32_t*>(&r1h);
    }
    stage_store_f16(stage, lane, h, g.out16, g.ldo, m_base, g.M, nb, g.N);
  } else if (EPI == EPI_F32) {
    if (stage) {
      float* st = reinterpret_cast<float*>(stage);
      const int piece = lane & 7;
      if (g.accumulate) {
#pragma unroll
        for (int s8 = 0; s8 < 8; ++s8) {                            // coalesced read of the old values: 4 rows x 128 B
          const int r = 4 * s8 + (lane >> 3), mr = wrow(m_base, r);
          float4 old = make_float4(0.f, 0.f, 0.f, 0.f);
          if (mr < g.M && nb + piece * 4 < g.N) old = *reinterpret_cast<const float4*>(g.out32 + (size_t)mr * g.ld32 + nb + piece * 4);
          *reinterpret_cast<float4*>(st + r * 36 + piece * 4) = old;
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaf(v[j], g.scale, st[lane * 36 + j]);
        __syncwarp();
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] *= g.scale;
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) *reinterpret_cast<float4*>(st + lane * 36 + q * 4) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
      __syncwarp();
#pragma unroll
      for (int s8 = 0; s8 < 8; ++s8) {
        const int r = 4 * s8 + (lane >> 3), mr = wrow(m_base, r);
        if (mr < g.M && nb + piece * 4 < g.N)
          *reinterpret_cast<float4*>(g.out32 + (size_t)mr * g.ld32 + nb + piece * 4) = *reinterpret_cast<const float4*>(st + r * 36 + piece * 4);
      }
      __syncwarp();
    } else if (m < g.M) {
      float* o = g.out32 + (size_t)m * g.ld32 + nb;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        if (nb + j < g.N) o[j] = (g.accumulate ? o[j] : 0.f) + v[j] * g.scale;
      }
    }
  } else if (stage && g.ldgn == 1) {
    // EPI_ATOMIC, unit column stride: a thread owns a ROW, so direct atomics would hit 32 different rows
    // per instruction.  Transpose 16 columns at a time through the per-warp tile ([32][17] floats) so
    // each reduction instruction covers two rows x 16 consecutive floats.
    float* stf = reinterpret_cast<float*>(stage);
    const int c = lane & 15, rsub = lane >> 4;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
#pragma unroll
      for (int j = 0; j < 16; ++j) stf[lane * 17 + j] = v[half * 16 + j] * g.scale;
      __syncwarp();
      const int n = nb + half * 16 + c;
      const bool n_in = n >= g.n_lo && n < g.n_valid, n_bias = n == g.ones_col && g.gbias != nullptr;
      if (n_in || n_bias) {
#pragma unroll 4
        for (int r2 = 0; r2 < 16; ++r2) {
          const int r = r2 * 2 + rsub, mrow = wrow(m_base, r);
          if (mrow < g.M) {
            const float val = stf[r * 17 + c];
            if (n_in) atomicAdd(g.gdst + (size_t)mrow * g.ldgd + n, val);
            else atomicAdd(g.gbias + mrow, val);
          }
        }
      }
      __syncwarp();
    }
  } else if (m < g.M) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int n = nb + j;
      if (n >= g.n_lo && n < g.n_valid) atomicAdd(g.gdst + (size_t)m * g.ldgd + (size_t)n * g.ldgn, v[j] * g.scale);
      else if (n == g.ones_col && g.gbias) atomicAdd(g.gbias + m, v[j] * g.scale);
    }
  }
}

template <int A_MN, int B_MN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_gemm_umma(const __grid_constant__ CUtensorMap mapA1, const __grid_constant__ CUtensorMap mapA2,
            const __grid_constant__ CUtensorMap mapB, GemmArgs g) {
  // Persistent: each CTA walks tiles  t = blockIdx.x, blockIdx.x + gridDim.x, ...  of the (z, m, n) tile space
  // (n fastest, so the N-tiles of one row block run back to back and share A in L2).
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE_BYTES);
  uint64_t* empty = full + NSTAGE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tiles_total = g.mt * g.nt * g.zt;
  const int k_total = g.K1 + g.K2;

  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], N_CWARPS); }
    ptx::mbar_init_fence();
  }
  __syncthreads();
  ptx::pdl_wait();                 // everything above overlapped the predecessor's tail (programmatic dependent launch)
  ptx::pdl_launch_dependents();

#define TILE_COORDS(T)                                                              \
  const int tz = (T) / (g.mt * g.nt), trem = (T) - tz * (g.mt * g.nt);              \
  const int m0 = (trem / g.nt) * BM, n0 = (trem % g.nt) * BN;                       \
  const int k_begin = g.ksplit > 0 ? tz * g.ksplit : 0;                             \
  const int k_end = g.ksplit > 0 ? min(k_total, k_begin + g.ksplit) : k_total;      \
  const int n_chunks = (k_end - k_begin + BK - 1) / BK;

  if (warp == N_CWARPS) {
    // ===================== TMA producer =====================
    if (ptx::elect_one()) {
      uint32_t cc = 0;                        // running chunk counter across tiles
      for (int t = blockIdx.x; t < n_tiles_total; t += gridDim.x) {
        TILE_COORDS(t)
        for (int c = 0; c < n_chunks; ++c, ++cc) {
          const int s = cc % NSTAGE;
          if (cc >= NSTAGE) ptx::mbar_wait(&empty[s], ((cc / NSTAGE) - 1) & 1);
          unsigned char* sa = smem + s * STAGE_BYTES;
          unsigned char* sb = sa + BM * BK * 2;
          ptx::mbar_arrive_expect_tx(&full[s], STAGE_BYTES);
          const int k = k_begin + c * BK;                     // global K position of this chunk
          // A: source 1 covers [0, K1), source 2 covers [K1, K1+K2); chunks never straddle (K1 % 64 == 0 or K2 == 0)
          const bool second = (g.K2 > 0) && (k >= g.K1);
          const CUtensorMap* ma = second ? &mapA2 : &mapA1;
          const int ka = second ? k - g.K1 : k;
          if (A_MN) { tma_load_2d(sa, ma, &full[s], m0, ka); tma_load_2d(sa + 8192, ma, &full[s], m0 + 64, ka); }   // dims (M, K)
          else      tma_load_2d(sa, ma, &full[s], ka, m0);                                                          // dims (K, M)
          const int kb = g.b_k0 + k;
          if (B_MN) { tma_load_2d(sb, &mapB, &full[s], n0, kb); tma_load_2d(sb + 8192, &mapB, &full[s], n0 + 64, kb); }
          else      tma_load_2d(sb, &mapB, &full[s], kb, n0);
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns columns 64 wg .. 64 wg + 63 of the tile =====================
    const int wg = warp >> 2, wq = warp & 3;
    unsigned char* scratch = smem + NSTAGE * STAGE_BYTES + 1024 + warp * EPI_SCRATCH;
    unsigned char* stage = (EPI == EPI_RELU_F16 || EPI == EPI_GATE_F16 || EPI == EPI_ATOMIC) ? scratch : nullptr;
    float d0[32], d1[32];                     // rows 0..63 / 64..127 of the tile
    uint32_t cc = 0;
    for (int t = blockIdx.x; t < n_tiles_total; t += gridDim.x) {
      TILE_COORDS(t)
      for (int c = 0; c < n_chunks; ++c, ++cc) {
        const int s = cc % NSTAGE;
        ptx::mbar_wait(&full[s], (cc / NSTAGE) & 1);
        const uint32_t sa = ptx::smem_u32(smem + s * STAGE_BYTES), sb = sa + BM * BK * 2 + wg * 8192;
        const int klen = min(BK, k_end - (k_begin + c * BK));
        ptx::wgmma_fence();
#pragma unroll 1
        for (int ks = 0; ks * 16 < klen; ++ks) {
          const uint32_t ao = A_MN ? ks * 2048 : ks * 32, bo = B_MN ? ks * 2048 : ks * 32;
          const uint64_t bd = desc_sw128(sb + bo, 16, 1024);
          const uint32_t acc = (c > 0 || ks > 0) ? 1u : 0u;
          ptx::wgmma_n64<A_MN, B_MN>(d0, desc_sw128(sa + ao, 16, 1024), bd, acc);
          ptx::wgmma_n64<A_MN, B_MN>(d1, desc_sw128(sa + 8192 + ao, 16, 1024), bd, acc);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if (lane == 0) ptx::mbar_arrive(&empty[s]);
      }
      float v[32];
      const int nb = n0 + wg * 64;
      if (nb < g.N) { frag_rows<0>(d0, d1, scratch, lane, v); epi_chunk<EPI>(g, v, m0 + 16 * wq, lane, nb, g.bias, stage); }
      if (nb + 32 < g.N) { frag_rows<1>(d0, d1, scratch, lane, v); epi_chunk<EPI>(g, v, m0 + 16 * wq, lane, nb + 32, g.bias, stage); }
    }
  }
#undef TILE_COORDS
}

// ---------------------------------------------------------------------------------------------
// Weight-stationary variant for the skinny GEMMs of the forward / dgrad passes:
//   D[M][N] = A[M][K] * B   with  M = all points (10^5..10^6),  N <= 256,  K <= 384.
// The generic kernel above re-streams A and B for every 128 x 128 tile.  Here each persistent CTA (one per SM)
//   * loads the WHOLE B operand (all N, all K: <= 192 KB) into shared memory once,
//   * streams only A through a deep TMA ring (16 KB stages),
//   * covers every output column of a 128-row block with its two consumer warpgroups: warpgroup g owns NB blocks of
//     64 columns starting at 64 NB g (NB = 1 for N <= 128, 2 for N <= 256), two wgmma.m64n64k16 per block and K step.
// ---------------------------------------------------------------------------------------------
constexpr int WS_THREADS = 32 * (N_CWARPS + 1);            // warps 0..7 consumers, 8 = TMA producer
constexpr int WS_SMEM = 232448;            // 227 KB: all of it
constexpr int WS_ASTAGE = BM * BK * 2;     // 16 KB
constexpr int WS_MAXCHUNK = 8, WS_MAXSTAGE = 8;

struct WsGeom { int nb_bytes, n_chunks, n_stage; };

template <int B_MN, int EPI, int NB>
__global__ void __launch_bounds__(WS_THREADS, 1)
k_gemm_ws(const __grid_constant__ CUtensorMap mapA1, const __grid_constant__ CUtensorMap mapA2,
          const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapB2, GemmArgs g, WsGeom geo) {
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* sB = smem;                                        // [n_chunks][nb_bytes]
  unsigned char* sA = smem + geo.n_chunks * geo.nb_bytes;          // [n_stage][16 KB]
  unsigned char* tail = sA + geo.n_stage * WS_ASTAGE;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);              // [WS_MAXSTAGE]
  uint64_t* empty = full + WS_MAXSTAGE;                            // [WS_MAXSTAGE]
  uint64_t* bfull = empty + WS_MAXSTAGE;                           // [WS_MAXCHUNK] B chunk landed
  float* sbias = reinterpret_cast<float*>(tail + 256);             // [256]
  unsigned char* sstage = tail + 256 + 1024;                       // [8 warps][EPI_SCRATCH]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int k_total = g.K1 + g.K2;

  if (tid == 0) {
    for (int s = 0; s < geo.n_stage; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], N_CWARPS); }
    for (int c = 0; c < geo.n_chunks; ++c) ptx::mbar_init(&bfull[c], 1);
    ptx::mbar_init_fence();
  }
  if (EPI == EPI_RELU_F16 && tid < 256) sbias[tid] = tid < g.N ? g.bias[tid] : 0.f;
  if (EPI == EPI_GATE_F16 && g.r1_row && tid < 256) sbias[tid] = tid < g.N ? g.r1_col[tid] : 0.f;
  __syncthreads();
  ptx::pdl_wait();                 // barrier init / bias staging (parameters: written launches ago) overlap the predecessor
  ptx::pdl_launch_dependents();

  if (warp == N_CWARPS) {
    // ===================== TMA producer: B once, then the A ring =====================
    if (ptx::elect_one()) {
      for (int c = 0; c < geo.n_chunks; ++c) {
        unsigned char* sb = sB + c * geo.nb_bytes;
        const bool b_second = g.b_two && c * BK >= g.K1;
        const CUtensorMap* mb = b_second ? &mapB2 : &mapB;
        const int kb = g.b_k0 + c * BK - (b_second ? g.K1 : 0);
        if (B_MN) {
          const int panels = (g.N + 63) / 64;
          ptx::mbar_arrive_expect_tx(&bfull[c], panels * 8192);
          for (int q = 0; q < panels; ++q) tma_load_2d(sb + q * 8192, mb, &bfull[c], q * 64, kb);       // dims (N, K)
        } else {
          const int boxes = (g.N + 127) / 128;
          ptx::mbar_arrive_expect_tx(&bfull[c], boxes * 16384);
          for (int q = 0; q < boxes; ++q) tma_load_2d(sb + q * 16384, mb, &bfull[c], kb, q * 128);      // dims (K, N)
        }
      }
      uint32_t cc = 0;
      for (int t = blockIdx.x; t < g.mt; t += gridDim.x) {
        const int m0 = t * BM;
        for (int c = 0; c < geo.n_chunks; ++c, ++cc) {
          const int s = cc % geo.n_stage;
          if (cc >= (uint32_t)geo.n_stage) ptx::mbar_wait(&empty[s], ((cc / geo.n_stage) - 1) & 1);
          ptx::mbar_arrive_expect_tx(&full[s], WS_ASTAGE);
          const int k = c * BK;
          const bool second = (g.K2 > 0) && (k >= g.K1);
          tma_load_2d(sA + s * WS_ASTAGE, second ? &mapA2 : &mapA1, &full[s], second ? k - g.K1 : k, m0);
        }
      }
    }
  } else {
    // ===================== consumers =====================
    const int wg = warp >> 2, wq = warp & 3;
    unsigned char* scratch = sstage + warp * EPI_SCRATCH;
    float d[NB][2][32];
    uint32_t cc = 0, it = 0;
    for (int t = blockIdx.x; t < g.mt; t += gridDim.x, ++it) {
      for (int c = 0; c < geo.n_chunks; ++c, ++cc) {
        const int s = cc % geo.n_stage;
        if (it == 0) ptx::mbar_wait(&bfull[c], 0);
        ptx::mbar_wait(&full[s], (cc / geo.n_stage) & 1);
        const uint32_t sa = ptx::smem_u32(sA + s * WS_ASTAGE), sb = ptx::smem_u32(sB + c * geo.nb_bytes);
        const int klen = min(BK, k_total - c * BK);
        ptx::wgmma_fence();
#pragma unroll 1
        for (int ks = 0; ks * 16 < klen; ++ks) {
          const uint32_t acc = (c > 0 || ks > 0) ? 1u : 0u;
          const uint64_t ad0 = desc_sw128(sa + ks * 32, 16, 1024), ad1 = desc_sw128(sa + 8192 + ks * 32, 16, 1024);
#pragma unroll
          for (int q = 0; q < NB; ++q) {
            const int col0 = (wg * NB + q) * 64;
            if (col0 < g.N) {                                     // warpgroup-uniform
              const uint64_t bd = desc_sw128(sb + (col0 >> 6) * 8192 + (B_MN ? ks * 2048 : ks * 32), 16, 1024);
              ptx::wgmma_n64<0, B_MN>(d[q][0], ad0, bd, acc);
              ptx::wgmma_n64<0, B_MN>(d[q][1], ad1, bd, acc);
            }
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if (lane == 0) ptx::mbar_arrive(&empty[s]);
      }
      const int m_base = t * BM + 16 * wq;
      float v[32];
#pragma unroll
      for (int q = 0; q < NB; ++q) {
        const int nb = (wg * NB + q) * 64;
        if (nb < g.N) { frag_rows<0>(d[q][0], d[q][1], scratch, lane, v); epi_chunk<EPI, true>(g, v, m_base, lane, nb, sbias, scratch, nullptr, sbias); }
        if (nb + 32 < g.N) { frag_rows<1>(d[q][0], d[q][1], scratch, lane, v); epi_chunk<EPI, true>(g, v, m_base, lane, nb + 32, sbias, scratch, nullptr, sbias); }
      }
    }
  }
}

// ---- host: tensor maps ----------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    void* p = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// fp16 matrix with `rows` rows of `cols` contiguous elements, row pitch `ld` elements.
//   mn_major = 0: the matrix is [rows = M or N][cols = K]   (K contiguous)   -> box (64 k, 128 rows)
//   mn_major = 1: the matrix is [rows = K][cols = M or N]   (MN contiguous)  -> box (64 mn, 64 k), two per stage
static bool make_operand_map(CUtensorMap* map, const void* base, long long rows, long long cols, long long ld, int mn_major) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)(mn_major ? BK : BM)};
  cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct Operand { const void* base; long long rows, cols, ld; };

template <int A_MN, int B_MN, int EPI>
static cudaError_t launch_gemm(const Operand& a1, const Operand& a2, const Operand& b, GemmArgs g, int m_tiles, int n_tiles,
                               int z, cudaStream_t st) {
  int dev = 0;
  cudaGetDevice(&dev);
  const cudaError_t e = smem_limit_once<k_gemm_umma<A_MN, B_MN, EPI>>(dev, GEMM_SMEM);
  if (e != cudaSuccess) return e;
  CUtensorMap mA1, mA2, mB;
  if (!make_operand_map(&mA1, a1.base, a1.rows, a1.cols, a1.ld, A_MN)) return cudaErrorInvalidValue;
  if (a2.base) { if (!make_operand_map(&mA2, a2.base, a2.rows, a2.cols, a2.ld, A_MN)) return cudaErrorInvalidValue; }
  else mA2 = mA1;
  if (!make_operand_map(&mB, b.base, b.rows, b.cols, b.ld, B_MN)) return cudaErrorInvalidValue;
  g.mt = m_tiles; g.nt = n_tiles; g.zt = z;
  const long long total = (long long)m_tiles * n_tiles * z;
  const int grid = (int)std::min<long long>(total, (long long)sm_count(dev));
  return launch_k(k_gemm_umma<A_MN, B_MN, EPI>, dim3(grid), dim3(GEMM_THREADS), GEMM_SMEM, st, mA1, mA2, mB, g);
}

// Weight-stationary launch (A K-major, single N tile).  Returns cudaErrorNotSupported when the shape does not fit
// (caller falls back to the generic kernel).
template <int B_MN, int EPI>
static cudaError_t launch_gemm_ws(const Operand& a1, const Operand& a2, const Operand& b, GemmArgs g, int m_tiles, cudaStream_t st,
                                  const Operand* b2 = nullptr) {
  const int K = g.K1 + g.K2;
  WsGeom geo;
  geo.nb_bytes = (g.N + 127) / 128 * 128 * 128;
  geo.n_chunks = (K + BK - 1) / BK;
  const int avail = WS_SMEM - 2048 - N_CWARPS * EPI_SCRATCH - geo.n_chunks * geo.nb_bytes;
  geo.n_stage = std::min(WS_MAXSTAGE, avail / WS_ASTAGE);
  if (g.N > 256 || geo.n_chunks > WS_MAXCHUNK || geo.n_stage < 3 || g.ksplit > 0 || (g.K2 > 0 && g.K1 % BK != 0))
    return cudaErrorNotSupported;
  int dev = 0;
  cudaGetDevice(&dev);
  auto kern = g.N > 128 ? k_gemm_ws<B_MN, EPI, 2> : k_gemm_ws<B_MN, EPI, 1>;
  const cudaError_t e = g.N > 128 ? smem_limit_once<k_gemm_ws<B_MN, EPI, 2>>(dev, WS_SMEM)
                                   : smem_limit_once<k_gemm_ws<B_MN, EPI, 1>>(dev, WS_SMEM);
  if (e != cudaSuccess) return e;
  CUtensorMap mA1, mA2, mB;
  if (!make_operand_map(&mA1, a1.base, a1.rows, a1.cols, a1.ld, 0)) return cudaErrorInvalidValue;
  if (a2.base) { if (!make_operand_map(&mA2, a2.base, a2.rows, a2.cols, a2.ld, 0)) return cudaErrorInvalidValue; }
  else mA2 = mA1;
  if (!make_operand_map(&mB, b.base, b.rows, b.cols, b.ld, B_MN)) return cudaErrorInvalidValue;
  CUtensorMap mB2 = mB;
  g.b_two = 0;
  if (b2) { if (!make_operand_map(&mB2, b2->base, b2->rows, b2->cols, b2->ld, B_MN)) return cudaErrorInvalidValue; g.b_two = 1; }
  g.mt = m_tiles; g.nt = 1; g.zt = 1;
  const int grid = std::min(m_tiles, sm_count(dev));
  return launch_k(kern, dim3(grid), dim3(WS_THREADS), WS_SMEM, st, mA1, mA2, mB, mB2, g, geo);
}

// forward / dgrad GEMMs: weight-stationary when the shape fits, generic otherwise
template <int B_MN, int EPI>
static cudaError_t launch_gemm_auto(const Operand& a1, const Operand& a2, const Operand& b, GemmArgs g, int m_tiles,
                                    int n_tiles, cudaStream_t st) {
  cudaError_t e = launch_gemm_ws<B_MN, EPI>(a1, a2, b, g, m_tiles, st);
  if (e == cudaErrorNotSupported) { (void)cudaGetLastError(); e = launch_gemm<0, B_MN, EPI>(a1, a2, b, g, m_tiles, n_tiles, 1, st); }
  return e;
}

}  // namespace lw
