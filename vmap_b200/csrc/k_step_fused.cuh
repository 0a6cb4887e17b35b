// K1: ONE launch per optimisation step for hidden = 32 (sm_90a: wgmma, bulk async copy, mbarrier).
//   mask counts (render_rays.py:68,86) -> PE -> MLP -> volume render -> losses -> backward
//   -> per-object gradient reduction in a fixed order -> AdamW + fp16 weight-image refresh
// fp16 operands / fp32 accumulate on wgmma.mma_async (m64nNk16, accumulators in registers), weights staged per object
// with one bulk async copy.  CTA = 256 threads = two warpgroups; a tile is up to 128 sample points (whole rays) and
// walks through 12 dependent MMA stages (6 forward, 6 backward): threads write the stage's operands -> fence + CTA
// barrier -> each warpgroup issues the stage's wgmmas for its 64 points and waits -> the hidden-layer epilogues run on
// the accumulator fragments in registers.  B (weights) always comes from shared memory.  A comes from REGISTERS (RS
// form) wherever it is a hidden activation or a gated dY of this warpgroup's own 64 points: an m64n32 fp32 fragment
// packed to f16x2 by the epilogue IS the A fragment of two k16 steps, so the next stage reads the epilogue's registers
// (the same fp16 values it also stores for the weight-gradient MMAs).  A stays in shared memory (SS form) for the
// embedding blocks, dhead and the weight-gradient MMAs (K = points of both warpgroups).  Shared-memory operand layout: no-swizzle
// 8x8 core matrices, an activation block is [feature-group (8 feats)][point][8 feats] halves -- the same bytes serve
// as a K-major A operand (forward / dgrad: M = points, K = features) and as an MN-major operand (wgrad: M or N =
// features, K = points).  Weight gradients accumulate in REGISTERS across all the tiles a CTA owns for an object (each
// warpgroup owns 64 of the up-to-128 feature rows of every gradient tile: 96 registers per thread).
//   * PE, the heads, the volume render and PE backward work one thread (pair) per point; the heads' 4 columns and the
//     144 embedding-gradient columns cross from the fragment layout to the point layout through shared memory;
//   * rays never straddle a warp (32/S rays per warp), so transmittance, the five rendered sums, the variance and
//     the backward suffix sum are warp-shuffle scans over the sample axis in registers;
//   * dY_l is not stored over h_l: one spare 8 KB block (Z) and the blocks whose readers have retired are rotated
//     (dYc->Z, dY4->HC, dY3->FC4, dY2->HC, dY1->FC3);
//   * both head weight gradients and both head bias gradients come out of ONE wgrad ([fc4 | emb2 | hc] x dhead);
//   * the PE-direction gradient dB = dproj^T [x y z] is a wgrad MMA too;
//   * K0 (mask counts) runs in the prologue, K2 (AdamW) per object as soon as the object is complete: every (CTA,
//     object) segment writes its gradient partial to its own row and then counts itself into the object's readiness
//     word.  A CTA that has run all its tiles claims finish chunks (object, float4 column range; object order) from a
//     ticket counter, issues the chunk's p / m / v loads, waits for the object's readiness word to reach its segment
//     count, adds the object's rows in segment order (bitwise reproducible whichever CTA runs the chunk -- no
//     floating-point atomics anywhere) and applies AdamW exactly as k_adamw does.  Training launches are cooperative:
//     a waiting CTA needs every CTA that still runs tiles resident.
//   * Updating an object while other CTAs still run tiles is safe because no CTA loads object b's weight image (its
//     only read of b's parameters) once all of b's segments have flushed: a CTA's copy of b's image completes before
//     its first tile of b, which is before its segment of b flushes.  The finish writes p / m / v and the image of b
//     only after all of b's segments are counted.
//
// Reference arithmetic: embedding.py:82-91, model.py:54-85, render_rays.py:4-96, loss.py:5-62, their autograd
// backward (train.py:293-324) and torch.optim.AdamW.step + zero_grad (train.py:325-326).
#pragma once
#include <string>
#include <cmath>
#include "common.cuh"
#include "k_step_fp32.cuh"
#include "umma_ptx.cuh"
#include "k_umma_image.cuh"     // column maps, weight-image layout, PE ladders, packed-half helpers (namespace um)

struct FusedExtra {
  float* partials;            // [(B + grid)][stride] per-(CTA, object) gradient partials, row = blockIdx + object
  unsigned int* finish_sync;  // [SY_OBJ + 2 * B] sync words (uf::SY_*), all but the skip flags re-armed by the last CTA
                              // to leave: an object's words sit at the same place whatever B is, so a launch with
                              // more objects never finds a skip flag in a readiness counter
  const int* counts_in;       // optional [B][4] external mask counts (ray-sharded iMAP: all-reduced by the caller)
  int* counts_pub;            // [B][4] scratch: otherwise CTA c counts objects c, c + grid, ... ONCE and publishes here
  int fuse_adam;              // 1: the finish applies AdamW; 0: it adds the reduced gradient into `grads`
  float* p; float* m; float* v;
  __half* image_out; const int* img_index; int img_halves;
  int* step_counter;          // optional [B] device step numbers (t = counter + 1, incremented here)
  float step_size, bc2_sqrt;  // host-computed bias corrections when step_counter == nullptr
  double lr, b1d, b2d;
  float log_b1, log_b2;       // ln(beta1), ln(beta2)
  const float2* bc_table;     // [bc_n] (1 - beta1^t, sqrt(1 - beta2^t)) built on the host in double precision, t = index
  int bc_n;
  float lr_wd, one_m_b1, b2, one_m_b2, eps;
  int guard_loss;
  int* status;
  float* loss_sum;            // optional: sum over objects of the weighted loss totals, written by the last CTA to leave
};

namespace uf {

constexpr int GT = 256, NT = 256, FGB = 2048;
// feature-group index of each 8-feature block inside a group's activation region.  Contiguity that the MMAs rely on:
// [FC1|FC2|E1] (mid1 bias row = E1's constant-1 column, cat_layer K = 128), [FC3|FC4|E2|HC] (mid2 / alpha bias rows =
// E2's constant-1 column, color_linear K = 80, heads wgrad M = [fc4 | emb2 | hc]).
constexpr int FG_DH = 0, FG_FC1 = 2, FG_FC2 = 6, FG_E1 = 10, FG_FC3 = 22, FG_FC4 = 26, FG_E2 = 30, FG_HC = 36, FG_Z = 40, FG_DPR = 44;
constexpr int FG_TOTAL = 47;
constexpr int ACT_BYTES = FG_TOTAL * FGB;                         // 96256
// Embedding-gradient tile (fp32): [36 blocks of 4 columns][128 points][4]: blocks 0..23 = d_emb1 (96 columns),
// 24..35 = d_emb2 (48 columns).  The warpgroups store their wgmma fragments here; PE backward reads a point's row.
constexpr int EG_BLOCKS = 36, EG_E2 = 24, EG_BYTES = EG_BLOCKS * FGB;
constexpr int HD_BYTES = 128 * 16;                                // heads tile: [128 points][alpha, r, g, b] fp32
constexpr int SM_ACT0 = 0, SM_EG = ACT_BYTES, SM_W = SM_EG + EG_BYTES, SM_HD = SM_W + um::IMG_BYTES, SM_MISC = SM_HD + HD_BYTES;
constexpr int MISC_BYTES = 512;
constexpr int SM_CNT = SM_MISC + MISC_BYTES;                      // int [B][3] mask counts
constexpr int SMEM_MAX = 232448;                                  // 227 KB: the most one block may have on sm_90
constexpr int SMEM_SLACK = 16;                                   // the launch's dynamic shared memory: SM_CNT + 12 B + slack
constexpr int MAX_OBJ_SMEM = (SMEM_MAX - SM_CNT - SMEM_SLACK) / 12;   // objects whose counts fit
constexpr float LS = um::LS, INV_LS = um::INV_LS;

struct Misc {
  uint64_t wbar;
  int on[3];
  int fin;
  unsigned int ticket[2];      // finish: the chunk claimed for this round and the next
  float step_size, bc2_sqrt;
  float lsum[4][4];
};
static_assert(sizeof(Misc) <= MISC_BYTES, "Misc");

// cvt + ReLU in one instruction
__device__ __forceinline__ uint32_t pack_relu_h2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// wgrad accumulator (block 0..4, feature row) -> (param index of out-column 0, stride per out-column), or -1
__device__ __forceinline__ int wg_base(const VmbLayout& L, int blk, int lane, int& ld) {
  ld = 1;
  switch (blk) {
    case 0: {                                   // A = E1: lanes = emb1 columns
      if (lane >= 96) return -1;
      const int j = um::emb1_col_to_j(lane);
      if (j == -2) return L.o_bin;
      if (j < 0) return -1;
      ld = VMB_E1; return L.o_Win + j;
    }
    case 1:                                     // A = [FC1 | FC2 | E1...]: lane 64 = constant 1
      if (lane < 32) { ld = 32; return L.o_Wm1 + lane; }
      return lane == 64 ? L.o_bm1 : -1;
    case 2: {                                   // A = [FC2 | E1]
      if (lane < 32) { ld = 32 + VMB_E1; return L.o_Wcat + lane; }
      const int j = um::emb1_col_to_j(lane - 32);
      if (j == -2) return L.o_bcat;
      if (j < 0) return -1;
      ld = 32 + VMB_E1; return L.o_Wcat + 32 + j;
    }
    case 3:                                     // A = [FC3 | FC4 | E2...]: lane 64 + 42 = constant 1
      if (lane < 32) { ld = 32; return L.o_Wm2 + lane; }
      return lane == 64 + 42 ? L.o_bm2 : -1;
    default: {                                  // A = [FC4 | E2]
      if (lane < 32) { ld = 32 + L.e2; return L.o_Wcl + lane; }
      if (lane >= 80) return -1;
      const int j2 = um::emb2_col_to_j2(lane - 32);
      if (j2 == -2) return L.o_bcl;
      if (j2 < 0) return -1;
      ld = 32 + L.e2; return L.o_Wcl + 32 + j2;
    }
  }
}

// ---- MMA issue: warpgroup-collective wgmma.  The CTA's two warpgroups split M: for the forward / dgrad GEMMs (M = points)
// warpgroup h owns points 64h .. 64h+63 of the tile, for the weight-gradient GEMMs (M = features) features 64h .. 64h+63
// of the A block.  Rows past the block's real features read neighbouring blocks (for the dB tile, the start of the
// embedding-gradient tile), possibly while the other warpgroup's epilogue rewrites them: a race on rows whose
// accumulators are never stored, and on no others.
struct Mma {
  uint32_t a16, w16;               // (activation base, weight base) >> 4
  int mh;                          // this warpgroup's M half

  // shared-memory matrix descriptor, no swizzle: start address, leading / stride byte offsets (all >> 4)
  static __device__ __forceinline__ uint64_t mk(uint32_t base16, uint32_t off, uint32_t lbo, uint32_t sbo) {
    const uint32_t lo = ((base16 + (off >> 4)) & 0x3FFFu) | ((lbo >> 4) << 16);
    return ((uint64_t)(sbo >> 4) << 32) | lo;
  }
  __device__ __forceinline__ uint64_t a_k(int fg, int ks) const { return mk(a16, fg * FGB + mh * 1024 + ks * 4096, 2048, 128); }   // K-major A: M = this half's points
  __device__ __forceinline__ uint64_t xa_mn(int fg, int ks) const { return mk(a16, (fg + 8 * mh) * FGB + ks * 256, 128, 2048); }  // MN-major A: M = this half's features, K = points
  __device__ __forceinline__ uint64_t xb_mn(int fg, int ks) const { return mk(a16, fg * FGB + ks * 256, 128, 2048); }             // MN-major B: N = features, K = points
  __device__ __forceinline__ uint64_t w_k(int off, int ks) const { return mk(w16, off + ks * 1024, 512, 128); }
  __device__ __forceinline__ uint64_t w16_k(int off, int ks) const { return mk(w16, off + ks * 512, 256, 128); }
  __device__ __forceinline__ uint64_t w_mn(int off, int ks) const { return mk(w16, off + ks * 256, 128, 512); }
  __device__ __forceinline__ uint64_t w16_mn(int off) const { return mk(w16, off, 128, 256); }

  // dW += X^T dY over the tile's 128 points: A = X block (features on M), B = dY block (features on N)
  __device__ __forceinline__ void wgrad32(float (&d)[16], int fgX, int fgDY) const {
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) ptx::wgmma_n32<1, 1>(d, xa_mn(fgX, ks), xb_mn(fgDY, ks), 1u);
  }
  __device__ __forceinline__ void wgrad16(float (&d)[8], int fgX, int fgDY) const {
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) ptx::wgmma_n16<1, 1>(d, xa_mn(fgX, ks), xb_mn(fgDY, ks), 1u);
  }
};

// Work partition: CTA c owns tiles [begin[c], begin[c+1]) of the global list (object-major).  Built on the host
// (fused_partition): a CTA whose range crosses an object boundary -- it pays a second flush / weight load / pipeline
// fill -- gets correspondingly fewer tiles, and the CTAs with the most tiles sit on the last objects.
constexpr int MAX_CTAS = 192;
// finish_sync words: [SY_TICKET] next finish chunk, [SY_DEPART] CTAs done, [SY_PUB] objects whose mask counts are
// published, [SY_EMPTY + 0..2] any-empty flags, then per object b: [SY_OBJ + 2b] segments whose partial row is out,
// [SY_OBJ + 2b + 1] skip flag (loss guard) of the step
constexpr int SY_TICKET = 0, SY_DEPART = 1, SY_PUB = 2, SY_EMPTY = 3, SY_OBJ = 6;
struct Ranges { int begin[MAX_CTAS + 1]; };

// Phase trace (TRACE instantiation only, vmb_step_trace): thread 0 of each warpgroup stamps clock64() into its own
// row of TR_STRIDE words, row = 2 * CTA + warpgroup.  Header: [0] kernel start, [1] prologue done, [2] last segment
// done, [3] finish start, [4] kernel end, [5] tiles run, [6] cycles in segment flushes, [7] segments, [8..11]
// %globaltimer (ns) at [0], [2], [3], [4], and in warpgroup 0's row only: [12] cycles waiting for other CTAs, [13]
// finish calls.  Then TR_NST stamps for each of the first TR_TILES tiles: [0] tile start and [k] the end of phase k
// (1..18: PE, in_layer, mid1, cat_layer, mid2, color_linear + alpha, out_color, heads transpose, render + loss, d_hc,
// d_fc4, d_fc3, d_fc2, d_fc1, d_emb, EG store, PE backward, dB).
constexpr int TR_HDR = 16, TR_NST = 20, TR_TILES = 64, TR_STRIDE = TR_HDR + TR_TILES * TR_NST;
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ int cta_of_tile(const Ranges& rg, int G, int tile) {        // largest c with begin[c] <= tile
  int lo = 0, hi = G - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (rg.begin[mid] <= tile) lo = mid; else hi = mid - 1; }
  return lo;
}

// a point's network input t and, for the PE's paired fp32 arithmetic (um::project4), each coordinate twice
struct PeIn {
  float3 t;
  uint64_t p0, p1, p2;
  __device__ __forceinline__ explicit PeIn(float3 v)
      : t(v), p0(um::pk2(v.x, v.x)), p1(um::pk2(v.y, v.y)), p2(um::pk2(v.z, v.z)) {}
};

// ---- The network on one tile as the training step (k_step_fused), the pose step (k_track_fused.cuh) and
// relocalisation scoring (k_reloc.cuh) run it: the tile's shared-memory blocks, the two thread layouts and the wgmma
// descriptors, with one copy of the positional embedding, the hidden-layer and dgrad epilogues, the embedding-gradient
// tile's stores and loads and the PE backward -- their operand layout and fp16 rounding points.
struct Tile {
  unsigned char* act;              // activation blocks (FG_*)
  unsigned char* eg;               // fp32 embedding-gradient tile (EG_*)
  float* hd;                       // heads tile: [128 points][alpha, r, g, b]
  const float* wf;                 // fp32 part of the weight image: biases, heads, PE directions
  const float* Bd;
  Mma mm;
  // point layout (PE, heads, render: one thread pair per point): point slot, direction half (= warpgroup) ...
  int p, hsel;
  // ... and accumulator-fragment layout (wgmma m64nN): this thread holds rows fr0 and fr0 + 8, columns 8j + 2 cq + {0, 1}
  int cq, fr0;

  // quad: this thread's warp within its warpgroup
  __device__ __forceinline__ Tile(unsigned char* act_, unsigned char* eg_, unsigned char* w, float* hd_, int quad)
      : act(act_), eg(eg_), hd(hd_), wf(reinterpret_cast<const float*>(w + um::IMG_F32)), Bd(wf + um::F_DIRS) {
    const int tid = threadIdx.x, lane = tid & 31;
    p = tid & 127; hsel = tid >> 7;
    cq = lane & 3; fr0 = 64 * hsel + 16 * quad + (lane >> 2);
    mm.a16 = ptx::smem_u32(act) >> 4;
    mm.w16 = ptx::smem_u32(w) >> 4;
    mm.mh = hsel;
  }

  // E0: positional embedding (embedding.py:82-91) of this thread's network input into E1 / E2, and this point's
  // dhead row zeroed (cols 4..15 stay zero; 0..3 are written after the render)
  __device__ __forceinline__ void embed(const PeIn& in) const {
    const float3 t = in.t;
    uint4* e1 = reinterpret_cast<uint4*>(act + FG_E1 * FGB + p * 16);
    uint4* e2 = reinterpret_cast<uint4*>(act + FG_E2 * FGB + p * 16);
    const int q0 = hsel ? 3 : 0, q1 = hsel ? 5 : 3;
    // software pipeline over the 4-direction chunks: the NEXT chunk's projections, range reduction and MUFU
    // sin / cos are issued before the CURRENT chunk's doubling recurrence, which hides their latency
    uint64_t s01, s23, c01, c23;
    {
      uint64_t pj01, pj23;
      um::project4(Bd, q0, in.p0, in.p1, in.p2, pj01, pj23);
      um::sincos4_x2(pj01, pj23, s01, s23, c01, c23);
    }
#pragma unroll 1
    for (int q = q0; q < q1; ++q) {                    // directions 4q .. 4q+3
      float sv[4][6];
      uint64_t ns01 = 0, ns23 = 0, nc01 = 0, nc23 = 0;
      if (q + 1 < q1) {
        uint64_t pj01, pj23;
        um::project4(Bd, q + 1, in.p0, in.p1, in.p2, pj01, pj23);
        um::sincos4_x2(pj01, pj23, ns01, ns23, nc01, nc23);
      }
      um::sin_doubling4_x2(s01, s23, c01, c23, sv);
      s01 = ns01; s23 = ns23; c01 = nc01; c23 = nc23;
      const uint4 ua = make_uint4(um::pack_h2(sv[0][0], sv[0][1]), um::pack_h2(sv[0][2], sv[0][3]), um::pack_h2(sv[1][0], sv[1][1]), um::pack_h2(sv[1][2], sv[1][3]));
      const uint4 ub = make_uint4(um::pack_h2(sv[2][0], sv[2][1]), um::pack_h2(sv[2][2], sv[2][3]), um::pack_h2(sv[3][0], sv[3][1]), um::pack_h2(sv[3][2], sv[3][3]));
      const uint4 uc = make_uint4(um::pack_h2(sv[0][4], sv[0][5]), um::pack_h2(sv[1][4], sv[1][5]), um::pack_h2(sv[2][4], sv[2][5]), um::pack_h2(sv[3][4], sv[3][5]));
      e1[(2 * q + 1) * 128] = ua; e1[(2 * q + 2) * 128] = ub; e2[q * 128] = uc;
    }
    if (hsel) {
      // direction 20 shares chunk 0 of emb1 with [1, x, y, z] and chunk 5 of emb2 with the const-1 column
      float s[6];
      um::sin_ladder(fmaf(Bd[2 * um::DIRS_PITCH + 20], t.z, fmaf(Bd[um::DIRS_PITCH + 20], t.y, Bd[20] * t.x)), s);
      const uint4 u0 = make_uint4(um::pack_h2(1.0f, t.x), um::pack_h2(t.y, t.z), um::pack_h2(s[0], s[1]), um::pack_h2(s[2], s[3]));
      const uint4 u5 = make_uint4(um::pack_h2(s[4], s[5]), um::pack_h2(1.0f, 0.f), 0u, 0u);
      e1[0] = u0;
      e2[5 * 128] = u5;
      e1[11 * 128] = make_uint4(0u, 0u, 0u, 0u);
      uint4* dh = reinterpret_cast<uint4*>(act + FG_DH * FGB + p * 16);
      dh[0] = make_uint4(0u, 0u, 0u, 0u); dh[128] = make_uint4(0u, 0u, 0u, 0u);
    }
  }

  // hidden-layer epilogue on the fragment: acc + bias -> ReLU -> fp16 into block fg (read back by the dgrad gates), and
  // into u: the A operand (ptx::wgmma_n32_rs) of the next stage's two k-steps over these 32 features
  __device__ __forceinline__ void epi_relu(const float (&v)[16], int bias_off, int fg, uint32_t (&u)[8]) const {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 bb = *reinterpret_cast<const float2*>(wf + bias_off + 8 * j + 2 * cq);
      unsigned char* dst = act + (fg + j) * FGB + fr0 * 16 + cq * 4;
      u[2 * j] = pack_relu_h2(v[4 * j] + bb.x, v[4 * j + 1] + bb.y);
      u[2 * j + 1] = pack_relu_h2(v[4 * j + 2] + bb.x, v[4 * j + 3] + bb.y);
      *reinterpret_cast<uint32_t*>(dst) = u[2 * j];
      *reinterpret_cast<uint32_t*>(dst + 128) = u[2 * j + 1];
    }
  }
  // dgrad epilogue: dY = (h > 0) * fp16(acc); h is read from its own block, dY goes into u (the A operand of the dgrad
  // GEMMs that read dY) and, under STORE (the training step), to block fg_out, whose readers have retired, for the
  // weight-gradient GEMMs
  template <bool STORE>
  __device__ __forceinline__ void epi_dgrad(const float (&v)[16], int fg_h, int fg_out, uint32_t (&u)[8]) const {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int off = j * FGB + fr0 * 16 + cq * 4;
      const uint32_t h0 = *reinterpret_cast<const uint32_t*>(act + fg_h * FGB + off);
      const uint32_t h1 = *reinterpret_cast<const uint32_t*>(act + fg_h * FGB + off + 128);
      u[2 * j] = um::gate_h2(um::pack_h2(v[4 * j], v[4 * j + 1]), h0);
      u[2 * j + 1] = um::gate_h2(um::pack_h2(v[4 * j + 2], v[4 * j + 3]), h1);
      if constexpr (STORE) {
        *reinterpret_cast<uint32_t*>(act + fg_out * FGB + off) = u[2 * j];
        *reinterpret_cast<uint32_t*>(act + fg_out * FGB + off + 128) = u[2 * j + 1];
      }
    }
  }
  // embedding-gradient fragment (8-column groups starting at 4-column block blk0) -> the shared fp32 tile
  template <int N>
  __device__ __forceinline__ void eg_store(const float (&v)[N], int blk0) const {
#pragma unroll
    for (int j = 0; j < N / 4; ++j) {
      float* d = reinterpret_cast<float*>(eg + (blk0 + 2 * j + (cq >> 1)) * FGB + fr0 * 16 + (cq & 1) * 8);
      *reinterpret_cast<float2*>(d) = make_float2(v[4 * j], v[4 * j + 1]);
      *reinterpret_cast<float2*>(d + 32) = make_float2(v[4 * j + 2], v[4 * j + 3]);
    }
  }
  // eight consecutive embedding-gradient columns of this thread's point
  __device__ __forceinline__ void eg_load8(int blk, float (&o)[8]) const {
    const float4 u0 = *reinterpret_cast<const float4*>(eg + blk * FGB + p * 16);
    const float4 u1 = *reinterpret_cast<const float4*>(eg + (blk + 1) * FGB + p * 16);
    o[0] = u0.x; o[1] = u0.y; o[2] = u0.z; o[3] = u0.w; o[4] = u1.x; o[5] = u1.y; o[6] = u1.z; o[7] = u1.w;
  }

  // PE backward from the eg tile: dproj_d = pi * sum_k 2^k g_{k,d} cos(pi 2^k proj_d) for this warpgroup's directions
  // (hsel 0: 0..11, hsel 1: 12..20), under DPROJ written as the fp16 dproj block (A of the dB wgrad).  Returns this
  // warpgroup's half of the point's dL/dt = INV_LS (dE_xyz + sum_d dproj_d B_d) in fp32 (the rule of k_tlw_pose),
  // summed in a fixed order: hsel 0 dE_xyz, then directions 0..11; hsel 1 directions 12..20.  A caller that does not
  // read it does not compute it.  The pose tile has no dproj block (DPROJ = false).
  template <bool DPROJ>
  __device__ __forceinline__ float3 pe_backward(const PeIn& in) const {
    const float3 t = in.t;
    const int q0 = hsel ? 3 : 0, q1 = hsel ? 5 : 3;
    float jt0 = 0.f, jt1 = 0.f, jt2 = 0.f;
    if (!hsel) {                                      // emb1 cols 1..3 = d/d[x y z]
      const float4 e0 = *reinterpret_cast<const float4*>(eg + p * 16);
      jt0 = e0.y * INV_LS; jt1 = e0.z * INV_LS; jt2 = e0.w * INV_LS;
    }
    uint64_t c01, c23;
    {
      uint64_t pj01, pj23;
      um::project4(Bd, q0, in.p0, in.p1, in.p2, pj01, pj23);
      um::cos4_x2(pj01, pj23, c01, c23);
    }
#pragma unroll 1
    for (int q = q0; q < q1; ++q) {
      float g1a[8], g1b[8], g2[8];
      eg_load8(4 * q + 2, g1a);                      // emb1 cols of directions 4q, 4q+1 (k = 0..3)
      eg_load8(4 * q + 4, g1b);                      //                          4q+2, 4q+3
      eg_load8(EG_E2 + 2 * q, g2);                   // emb2 cols (k = 4, 5)
      float cv[4][6], dp[4];
      uint64_t nc01 = 0, nc23 = 0;
      if (q + 1 < q1) {                              // next chunk's front half before this chunk's recurrence
        uint64_t pj01, pj23;
        um::project4(Bd, q + 1, in.p0, in.p1, in.p2, pj01, pj23);
        um::cos4_x2(pj01, pj23, nc01, nc23);
      }
      um::cos_doubling4_x2(c01, c23, cv);
      c01 = nc01; c23 = nc23;
#pragma unroll
      for (int dd = 0; dd < 4; ++dd) {
        const float* g1 = (dd < 2) ? (g1a + dd * 4) : (g1b + (dd - 2) * 4);
        float d = g1[0] * cv[dd][0];
        d = fmaf(2.f * g1[1], cv[dd][1], d);
        d = fmaf(4.f * g1[2], cv[dd][2], d);
        d = fmaf(8.f * g1[3], cv[dd][3], d);
        d = fmaf(16.f * g2[dd * 2], cv[dd][4], d);
        d = fmaf(32.f * g2[dd * 2 + 1], cv[dd][5], d);
        dp[dd] = d * VMB_PI_F;
        const int dir = 4 * q + dd;
        const float g = dp[dd] * INV_LS;
        jt0 = fmaf(g, Bd[dir], jt0); jt1 = fmaf(g, Bd[um::DIRS_PITCH + dir], jt1); jt2 = fmaf(g, Bd[2 * um::DIRS_PITCH + dir], jt2);
      }
      // directions 4q..4q+3 = columns (4q)%8.. of feature group q/2
      if constexpr (DPROJ)
        *reinterpret_cast<uint2*>(act + (FG_DPR + (q >> 1)) * FGB + p * 16 + (q & 1) * 8) =
            make_uint2(um::pack_h2(dp[0], dp[1]), um::pack_h2(dp[2], dp[3]));
    }
    if (hsel) {                                       // direction 20: emb1 cols 4..7, emb2 cols 40, 41
      float g1[8], g2[8], c[6];
      eg_load8(0, g1);
      eg_load8(EG_E2 + 10, g2);
      um::cos_ladder(fmaf(Bd[2 * um::DIRS_PITCH + 20], t.z, fmaf(Bd[um::DIRS_PITCH + 20], t.y, Bd[20] * t.x)), c);
      float d = g1[4] * c[0];
      d = fmaf(2.f * g1[5], c[1], d); d = fmaf(4.f * g1[6], c[2], d); d = fmaf(8.f * g1[7], c[3], d);
      d = fmaf(16.f * g2[0], c[4], d); d = fmaf(32.f * g2[1], c[5], d);
      if constexpr (DPROJ)
        *reinterpret_cast<uint2*>(act + (FG_DPR + 2) * FGB + p * 16 + 8) = make_uint2(um::pack_h2(d * VMB_PI_F, 0.f), 0u);
      const float g = (d * VMB_PI_F) * INV_LS;
      jt0 = fmaf(g, Bd[20], jt0); jt1 = fmaf(g, Bd[um::DIRS_PITCH + 20], jt1); jt2 = fmaf(g, Bd[2 * um::DIRS_PITCH + 20], jt2);
    }
    return make_float3(jt0, jt1, jt2);
  }
};

}  // namespace uf

// ---------------------------------------------------------------------------------------------------------------
// JOINT (the joint map-and-pose step, vmb_joint_step_fused): the PE backward also forms each point's pose gradient
// dL/dt = INV_LS (dE_xyz + sum_d dproj_d B_d) in fp32 from the same cosines and the same pre-update directions Bd as the
// dB wgrad (the rule of k_tlw_pose).  Each warpgroup sums its own directions (hsel 0: dE_xyz, then 0..11; hsel 1:
// 12..20) and stores its half to jdt[b][point][hsel][3] (fp32, plain stores); k_joint_rows adds the halves in that
// order.  jdt is read only under JOINT: the plain instantiations compile to the same SASS as without it.
// Registers (ptxas -v, sm_90a), no spills: JOINT S = any / 10 / 14: 249 / 249 / 249 (plain: 251 / 251 / 251; TRACE
// S = 10: 252).
// TRACE (phase-stamped build, S = 10 only): `trace` as uf::TR_STRIDE describes; the other instantiations ignore it and
// contain no trace code.
template <int SC, bool JOINT, bool TRACE = false>
__global__ void __launch_bounds__(uf::NT, 1)
k_step_fused(StepParams a, FusedExtra x, VmbLayout L, const unsigned char* image, const __grid_constant__ uf::Ranges rg, int tpo, int nr, int rpw,
             float* jdt, unsigned long long* trace) {
  using namespace uf;
  extern __shared__ __align__(1024) unsigned char smem[];
  Misc* misc = reinterpret_cast<Misc*>(smem + SM_MISC);
  int* cnt = reinterpret_cast<int*>(smem + SM_CNT);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S = SC ? SC : a.S, R = a.R;
  unsigned long long* tr = nullptr;
  const bool tr_on = TRACE && (tid & 127) == 0;
  int tr_t = 0, tr_nseg = 0;
  long long tr_flush = 0, tr_f0 = 0;
  if constexpr (TRACE) tr = trace + (size_t)(2 * blockIdx.x + (tid >> 7)) * TR_STRIDE;
  long long tr_wait = 0;
  int tr_calls = 0;
#define TR_STAMP(slot) do { if constexpr (TRACE) { if (tr_on) tr[slot] = clock64(); } } while (0)
#define TR_STAMP2(slot, gslot) do { if constexpr (TRACE) { if (tr_on) { tr[slot] = clock64(); tr[gslot] = globaltimer(); } } } while (0)
#define TR_TILE(k) do { if constexpr (TRACE) { if (tr_on && tr_t < TR_TILES) tr[TR_HDR + tr_t * TR_NST + (k)] = clock64(); } } while (0)
  TR_STAMP2(0, 8);

  if (tid == 0) {
    ptx::mbar_init(&misc->wbar, 1);
    misc->on[0] = misc->on[1] = misc->on[2] = 1;
    ptx::mbar_init_fence();
  }
  const int G = gridDim.x;
  const long long gt_begin = rg.begin[blockIdx.x], gt_end = rg.begin[blockIdx.x + 1];
  __syncthreads();
  if (tid == 0 && gt_begin < gt_end) {     // first object's weight image: in flight while the mask counts run
    ptx::mbar_arrive_expect_tx(&misc->wbar, um::IMG_BYTES);
    ptx::bulk_g2s(smem + SM_W, image + (size_t)(gt_begin / tpo) * um::IMG_BYTES, um::IMG_BYTES, &misc->wbar);
  }
  // ---- K0 in the prologue: mask counts of EVERY object (the any-empty early-out couples them, render_rays.py:68-73).
  // Training launch without counts_in: CTA c counts objects c, c + grid, ... ONCE and publishes counts + empty flags +
  // a "published" counter in global memory; every CTA starts its tiles at once and acquires the counts right before
  // its first volume render (thousands of cycles later: the wait is free).  With counts_in, every CTA copies them.
  const bool pub_counts = !x.counts_in && !a.fwd_only;
  unsigned int* gbar = x.finish_sync;                   // words as uf::SY_* describes
  if (pub_counts) {
    for (int b = blockIdx.x; b < a.B; b += G) {
      if (tid < 3) cnt[tid] = 0;
      __syncthreads();
      const unsigned char* s = a.sem + (size_t)b * a.sem_stride;
      const unsigned char* m = a.mask + (size_t)b * a.mask_stride;
      const bool vec = (((size_t)s | (size_t)m) & 3) == 0;
      const int nw = vec ? (R >> 2) : 0;
      // one bit per byte: nonzero(x) folds a byte's bits into bit 0 (labels are 0 / 1 / 2, masks any nonzero = true)
      auto nzb = [](uint32_t v) { v |= v >> 4; v |= v >> 2; v |= v >> 1; return v & 0x01010101u; };
      int nd = 0, no = 0, ns = 0;
      for (int w = tid; w < nw; w += NT) {               // four rays per 32-bit load
        const uint32_t sv = __ldg(reinterpret_cast<const uint32_t*>(s) + w), mv = __ldg(reinterpret_cast<const uint32_t*>(m) + w);
        const uint32_t o = nzb(sv);
        no += __popc(o); nd += __popc(o & nzb(mv)); ns += __popc(nzb(sv ^ 0x02020202u));
      }
      for (int r = (nw << 2) + tid; r < R; r += NT) {
        const int sv = s[r], mo = sv != 0;
        nd += (m[r] != 0) & mo; no += mo; ns += sv != 2;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        nd += __shfl_xor_sync(0xffffffffu, nd, o); no += __shfl_xor_sync(0xffffffffu, no, o); ns += __shfl_xor_sync(0xffffffffu, ns, o);
      }
      if (lane == 0) { atomicAdd(&cnt[0], nd); atomicAdd(&cnt[1], no); atomicAdd(&cnt[2], ns); }
      __syncthreads();
      if (tid == 0) {
        for (int k = 0; k < 3; ++k) {
          x.counts_pub[b * 4 + k] = cnt[k];
          if (cnt[k] == 0) atomicOr(&gbar[SY_EMPTY + k], 1u);
        }
        __threadfence();
        atomicAdd(&gbar[SY_PUB], 1u);
      }
      __syncthreads();
    }
  } else if (!a.fwd_only) {                             // counts_in given
    for (int i = tid; i < a.B * 3; i += NT) {
      const int c = x.counts_in[(i / 3) * 4 + (i % 3)];
      cnt[i] = c;
      if (c == 0) misc->on[i % 3] = 0;
    }
  }
  __syncthreads();
  TR_STAMP(1);

  uint32_t wpar = 0;                  // weight-barrier parity (one completion per segment)

  // thread roles: point layout (PE, heads, render: one thread pair per point) ...
  const int p = tid & 127, hsel = tid >> 7;               // point slot, direction half (= warpgroup)
  const int quad = (warp & 3);
  const int rw = lane / S, sidx = lane - rw * S;        // ray of this warp, sample index
  const bool lane_used = rw < rpw;
  const int ray_in_tile = quad * rpw + rw;
  const int seg_lo = lane - sidx;                        // first lane of this ray
  unsigned char* act = smem + SM_ACT0;
  unsigned char* eg = smem + SM_EG;
  float* hd = reinterpret_cast<float*>(smem + SM_HD);
  const float* wf = reinterpret_cast<const float*>(smem + SM_W + um::IMG_F32);
  // ... and accumulator-fragment layout (wgmma m64nN): this thread holds rows fr0 and fr0 + 8, columns 8j + 2 cq + {0, 1}
  const int cq = lane & 3, fr0 = 64 * hsel + 16 * quad + (lane >> 2);
  Mma mm;
  mm.a16 = ptx::smem_u32(act) >> 4;
  mm.w16 = ptx::smem_u32(smem + SM_W) >> 4;
  mm.mh = hsel;
  const Tile tl(act, eg, smem + SM_W, hd, quad);
  // persistent weight-gradient accumulators of the current object (this warpgroup's 64 feature rows)
  float wIN[16] = {}, wM1[16] = {}, wCAT[16] = {}, wM2[16] = {}, wCL[16] = {}, wHD[8] = {}, wDB[8] = {};
  // loss weights of this thread's current object: (term enabled: no object has an empty mask) / (this object's mask count)
  const float on_d = misc->on[0] ? 1.f : 0.f, on_c = misc->on[1] ? 1.f : 0.f, on_o = misc->on[2] ? 1.f : 0.f;
  float w_d = 0.f, w_c = 0.f, w_o = 0.f;
  bool cnt_ready = !pub_counts;       // published counts acquired?

  for (long long gt = gt_begin; gt < gt_end;) {
    const int b = (int)(gt / tpo);
    const int t0 = (int)(gt - (long long)b * tpo);
    const int t1 = (int)min((long long)tpo, (long long)t0 + (gt_end - gt));   // this segment's tiles of object b
    gt += t1 - t0;

    // ---- this object's weight image (one bulk copy global -> shared, issued before the previous segment's flush) ----
    um::mbar_wait_or_trap(&misc->wbar, wpar);
    wpar ^= 1;

    float ls_d = 0.f, ls_c = 0.f, ls_o = 0.f;
    {
    const float isc = 1.0f / a.scale[b];
    bool seg_w = false;               // published counts: w_d / w_c / w_o hold this segment's object?
    if (x.counts_in && !a.fwd_only) {
      w_d = on_d / ((float)cnt[b * 3 + 0] + 1e-10f);
      w_c = on_c / ((float)cnt[b * 3 + 1] + 1e-10f);
      w_o = on_o / ((float)cnt[b * 3 + 2] + 1e-10f);
    }

    // A stage: operands written by generic stores -> fence for the async proxy -> CTA barrier -> each warpgroup issues
    // the stage's wgmmas on its M half and, behind them, the layer's weight-gradient wgmmas into the persistent
    // accumulators -> commit -> wait.
#define OPERANDS_READY() do { ptx::fence_async_smem(); __syncthreads(); ptx::wgmma_fence(); } while (0)
#define MMA_DONE() do { ptx::wgmma_commit(); ptx::wgmma_wait<0>(); } while (0)
    // prefetched inputs of the next tile (global-load latency overlaps the current tile)
    float nx = 0.f, ny = 0.f, nz = 0.f, nzv = 0.f, n_gd = 0.f, n_c0 = 0.f, n_c1 = 0.f, n_c2 = 0.f;
    // (nothing computes on the loaded values here: the first use of a load stalls the warp for the memory latency)
    int n_sem = 0, n_msk = 0;
    bool n_live = false;
    // this object's base pointers, formed once per segment (the kernel-parameter loads and 64-bit stride products
    // otherwise sit, with their latencies, in every tile's prefetch)
    const float* pcs_b = a.pcs + (size_t)b * a.pcs_stride + (size_t)sidx * 3;
    const float* z_b = a.z + (size_t)b * a.z_stride + sidx;
    const float* gd_b = a.gt_depth + (size_t)b * a.gt_depth_stride;
    const float* gc_b = a.gt_colour + (size_t)b * a.gt_colour_stride;
    const unsigned char* sem_b = a.sem + (size_t)b * a.sem_stride;
    const unsigned char* msk_b = a.mask + (size_t)b * a.mask_stride;
    const bool want_targets = hsel == 0 && !a.fwd_only;
    auto prefetch = [&](int t) {
      nx = ny = nz = nzv = 0.f; n_gd = n_c0 = n_c1 = n_c2 = 0.f; n_sem = 0; n_msk = 0; n_live = false;
      if (t >= t1 || !lane_used) return;
      const int ray = t * nr + ray_in_tile;
      if (ray >= R) return;
      const size_t pi = (size_t)ray * S;
      const float* pp = pcs_b + pi * 3;
      nx = pp[0]; ny = pp[1]; nz = pp[2];
      if (want_targets) {                               // the render / loss lanes: every lane of a ray reads the ray's targets
        nzv = z_b[pi];
        n_gd = gd_b[ray];
        const float* gcp = gc_b + (size_t)ray * 3;
        n_c0 = gcp[0]; n_c1 = gcp[1]; n_c2 = gcp[2];
        n_sem = sem_b[ray];
        n_msk = msk_b[ray];
      }
      n_live = true;                                      // live point
    };
    prefetch(t0);

    for (int t = t0; t < t1; ++t) {
      TR_TILE(0);
      const int ray = t * nr + ray_in_tile;
      // ---- E0: positional embedding (embedding.py:82-91) ----------------------------------------------------
      const float t0x = nx * isc, t1x = ny * isc, t2x = nz * isc, zv = nzv;
      const PeIn tin(make_float3(t0x, t1x, t2x));
      const float gd = n_gd, gc0 = n_c0, gc1 = n_c1, gc2 = n_c2;
      const int sv = n_sem, mv = n_msk;
      const bool live = n_live;
      prefetch(t + 1);
      tl.embed(tin);
      TR_TILE(1);
      float acc[16], hacc[8];
      uint32_t ua[8];                                   // the last epilogue's fp16 output: A of the next stage (RS)
      OPERANDS_READY();                                 // in_layer: emb1 (K = 96)
#pragma unroll
      for (int ks = 0; ks < 6; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_E1, ks), mm.w_k(um::IMG_WIN, ks), ks > 0);
      MMA_DONE();
      tl.epi_relu(acc, um::F_BIN, FG_FC1, ua);
      TR_TILE(2);
      OPERANDS_READY();                                 // mid1: fc1
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, mm.w_k(um::IMG_WM1, ks), ks > 0);
      MMA_DONE();
      tl.epi_relu(acc, um::F_BM1, FG_FC2, ua);
      TR_TILE(3);
      OPERANDS_READY();                                 // cat_layer: [fc2 | emb1] (K = 128)
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, mm.w_k(um::IMG_WCAT, ks), ks > 0);
#pragma unroll
      for (int ks = 2; ks < 8; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_FC2, ks), mm.w_k(um::IMG_WCAT, ks), 1u);
      MMA_DONE();
      tl.epi_relu(acc, um::F_BCAT, FG_FC3, ua);
      TR_TILE(4);
      OPERANDS_READY();                                 // mid2: fc3
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, mm.w_k(um::IMG_WM2, ks), ks > 0);
      MMA_DONE();
      tl.epi_relu(acc, um::F_BM2, FG_FC4, ua);
      TR_TILE(5);
      OPERANDS_READY();                                 // color_linear: [fc4 | emb2] (K = 80) ; out_alpha: fc4 -> column 0
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, mm.w_k(um::IMG_WCL, ks), ks > 0);
#pragma unroll
      for (int ks = 2; ks < 5; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_FC4, ks), mm.w_k(um::IMG_WCL, ks), 1u);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16_rs<0>(hacc, ua + 4 * ks, mm.w16_k(um::IMG_WA16, ks), ks > 0);
      MMA_DONE();
      tl.epi_relu(acc, um::F_BCL, FG_HC, ua);
      if (cq == 0) { hd[fr0 * 4] = hacc[0]; hd[(fr0 + 8) * 4] = hacc[2]; }
      TR_TILE(6);
      OPERANDS_READY();                                 // out_color: hc -> columns 1..3
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16_rs<0>(hacc, ua + 4 * ks, mm.w16_k(um::IMG_WOC16, ks), ks > 0);
      MMA_DONE();
      if (cq == 0) { hd[fr0 * 4 + 1] = hacc[1]; hd[(fr0 + 8) * 4 + 1] = hacc[3]; }
      if (cq == 1) { hd[fr0 * 4 + 2] = hacc[0]; hd[fr0 * 4 + 3] = hacc[1]; hd[(fr0 + 8) * 4 + 2] = hacc[2]; hd[(fr0 + 8) * 4 + 3] = hacc[3]; }
      TR_TILE(7);
      __syncthreads();                                  // heads tile: fragment layout -> point layout
      TR_TILE(8);
      // ---- heads + volume render + losses + ray gradients, all in registers of the hsel == 0 warps ---------------
      // rays never straddle a warp: the scans over the sample axis are warp shuffles
      auto raysum = [&](float v) {                      // per-ray sum: guarded tree reduction to the ray's first lane, broadcast
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          if (off < S) { const float u = __shfl_down_sync(0xffffffffu, v, off); if (sidx + off < S) v += u; }
        }
        return __shfl_sync(0xffffffffu, v, seg_lo);
      };
      float araw = 0.f, occ = 0.f, fr = 1.f, Tr = 1.f, w = 0.f, D = 0.f, O = 0.f, V = 0.f;
      if (hsel == 0) {
        if (pub_counts && !seg_w) {                     // acquire the published mask counts (first render only)
          if (!cnt_ready) {
            const volatile unsigned int* pubd = gbar + SY_PUB;
            unsigned int spins = 0;
            while (*pubd < (unsigned int)a.B) { if (++spins > 2000000000u) __trap(); }
            __threadfence();
            cnt_ready = true;
          }
          const volatile unsigned int* ef = gbar + SY_EMPTY;
          const volatile int* cp = x.counts_pub + b * 4;
          w_d = (ef[0] ? 0.f : 1.f) / ((float)cp[0] + 1e-10f);
          w_c = (ef[1] ? 0.f : 1.f) / ((float)cp[1] + 1e-10f);
          w_o = (ef[2] ? 0.f : 1.f) / ((float)cp[2] + 1e-10f);
          seg_w = true;
        }
        araw = (hd[p * 4] + wf[um::F_BA]) * 10.0f;                                   // model.py:77
        occ = um::fast_sigmoid(araw);                                            // render_rays.py:6
        if (!a.fwd_only) {
          if (!live) occ = 0.f;
          // termination: T_s = prod_{j<s} (1 - occ_j + 1e-10) (render_rays.py:29), inclusive scan then shift
          fr = 1.f - occ + 1e-10f;
          float inc = fr;
#pragma unroll
          for (int off = 1; off < 32; off <<= 1) {
            if (off < S) { const float u = __shfl_up_sync(0xffffffffu, inc, off); if (sidx >= off) inc *= u; }
          }
          Tr = __shfl_up_sync(0xffffffffu, inc, 1);
          if (sidx == 0) Tr = 1.f;
          w = occ * Tr;                                                           // render_rays.py:34
          D = raysum(w * zv); O = raysum(w);
          const float dz = zv - D;
          V = raysum(w * dz * dz);                                                // render_rays.py:47-51 (detached)
        }
      }
      if (hsel == 0) {
        const float4 hv = *reinterpret_cast<const float4*>(hd + p * 4);
        const float c0 = um::fast_sigmoid(hv.y + wf[um::F_BOC + 0]), c1 = um::fast_sigmoid(hv.z + wf[um::F_BOC + 1]),
                    c2 = um::fast_sigmoid(hv.w + wf[um::F_BOC + 2]);
        if (a.fwd_only) {                               // eval_points (trainer.py:77-90): raw alpha*10, sigmoid colour per point
          if (live) {
            const size_t n = (size_t)ray * S + sidx;
            a.out_alpha[(size_t)b * a.alpha_stride + n] = araw;
            float* oc = a.out_colour + (size_t)b * a.colour_stride + n * 3;
            oc[0] = c0; oc[1] = c1; oc[2] = c2;
          }
        } else {
          const float C0 = raysum(w * c0), C1 = raysum(w * c1), C2 = raysum(w * c2);
          const float m_o = (live && sv != 0) ? 1.f : 0.f, m_s = (live && sv != 2) ? 1.f : 0.f, m_d = (mv != 0) ? m_o : 0.f;
          const float info = 1.f / (sqrtf(V) + 1e-4f);                            // render_rays.py:74-79
          const float e_d = D - gd, e_o = O - m_o, e_c0 = C0 - gc0, e_c1 = C1 - gc1, e_c2 = C2 - gc2;
          if (live && sidx == 0) {
            if (a.r_depth) a.r_depth[(size_t)b * R + ray] = D;
            if (a.r_var) a.r_var[(size_t)b * R + ray] = V;
            if (a.r_opacity) a.r_opacity[(size_t)b * R + ray] = O;
            if (a.r_colour) { float* rc = a.r_colour + ((size_t)b * R + ray) * 3; rc[0] = C0; rc[1] = C1; rc[2] = C2; }
            ls_d += w_d * fabsf(e_d) * m_d * info;
            ls_c += w_c * (fabsf(e_c0) + fabsf(e_c1) + fabsf(e_c2)) * m_o;
            ls_o += w_o * fabsf(e_o) * m_s;
          }
          if (a.backward) {
            const float gD = LS * w_d * vmb_sign(e_d) * m_d * info;
            const float kc = LS * w_c * a.cs * m_o;
            const float gC0 = kc * vmb_sign(e_c0), gC1 = kc * vmb_sign(e_c1), gC2 = kc * vmb_sign(e_c2);
            const float gO = LS * w_o * a.os * vmb_sign(e_o) * m_s;
            // d(loss)/d(occ_s) through the termination product: G_s T_s - (sum_{k>s} G_k w_k) / (1 - occ_s + 1e-10)
            const float Gs = fmaf(gD, zv, fmaf(gC0, c0, fmaf(gC1, c1, fmaf(gC2, c2, gO))));
            float suf = Gs * w;                                                   // inclusive suffix scan
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
              if (off < S) { const float u = __shfl_down_sync(0xffffffffu, suf, off); if (sidx + off < S) suf += u; }
            }
            float sx = __shfl_down_sync(0xffffffffu, suf, 1);
            if (sidx + 1 >= S) sx = 0.f;
            const float docc = Gs * Tr - __fdividef(sx, fr);
            const float da = 10.0f * docc * occ * (1.f - occ);                    // model.py:77
            if (live)
              *reinterpret_cast<uint2*>(act + FG_DH * FGB + p * 16) =
                  make_uint2(um::pack_h2(da, gC0 * w * c0 * (1.f - c0)), um::pack_h2(gC1 * w * c1 * (1.f - c1), gC2 * w * c2 * (1.f - c2)));
          }
        }
      }
      TR_TILE(9);
      if (a.fwd_only || !a.backward) { __syncthreads(); continue; }
      // dgrad chain: A = dhead (point layout, written by the render) from shared memory, every gated dY from the
      // registers of the epilogue that made it; dYc and dY3 stay in registers until the d_emb stage reads them
      uint32_t uyc[8], uy3[8];
      OPERANDS_READY();                                 // d_hc = dhead @ W_oc ; heads wgrad (out_alpha + out_color, weights and biases)
      ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_DH, 0), mm.w16_mn(um::IMG_WOC16), 0u);
      mm.wgrad16(wHD, FG_FC4, FG_DH);
      MMA_DONE();
      tl.epi_dgrad<true>(acc, FG_HC, FG_Z, uyc);                 // dYc -> Z
      TR_TILE(10);
      OPERANDS_READY();                                 // d_fc4 = dYc @ W_cl[:, :32] + dhead @ W_a ; wgrad color_linear
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uyc + 4 * ks, mm.w_mn(um::IMG_WCL, ks), ks > 0);
      ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_DH, 0), mm.w16_mn(um::IMG_WA16), 1u);
      mm.wgrad32(wCL, FG_FC4, FG_Z);
      MMA_DONE();
      tl.epi_dgrad<true>(acc, FG_FC4, FG_HC, ua);                // dY4 -> HC
      TR_TILE(11);
      OPERANDS_READY();                                 // d_fc3 = dY4 @ W_m2 ; wgrad mid2
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, ua + 4 * ks, mm.w_mn(um::IMG_WM2, ks), ks > 0);
      mm.wgrad32(wM2, FG_FC3, FG_HC);
      MMA_DONE();
      tl.epi_dgrad<true>(acc, FG_FC3, FG_FC4, uy3);              // dY3 -> FC4
      TR_TILE(12);
      OPERANDS_READY();                                 // d_fc2 = dY3 @ W_cat[:, :32] ; wgrad cat_layer
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uy3 + 4 * ks, mm.w_mn(um::IMG_WCAT, ks), ks > 0);
      mm.wgrad32(wCAT, FG_FC2, FG_FC4);
      MMA_DONE();
      tl.epi_dgrad<true>(acc, FG_FC2, FG_HC, ua);                // dY2 -> HC
      TR_TILE(13);
      OPERANDS_READY();                                 // d_fc1 = dY2 @ W_m1 ; wgrad mid1
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, ua + 4 * ks, mm.w_mn(um::IMG_WM1, ks), ks > 0);
      mm.wgrad32(wM1, FG_FC1, FG_HC);
      MMA_DONE();
      tl.epi_dgrad<true>(acc, FG_FC1, FG_FC3, ua);               // dY1 -> FC3
      TR_TILE(14);
      // d_emb1 = dY3 @ W_cat[:, 32:] + dY1 @ W_in (32 columns at a time), d_emb2 = dYc @ W_cl[:, 32:] ; wgrad in_layer
      OPERANDS_READY();
#pragma unroll
      for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uy3 + 4 * ks, mm.w_mn(um::IMG_WCAT + (4 + 4 * c) * 512, ks), ks > 0);
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, ua + 4 * ks, mm.w_mn(um::IMG_WIN + 4 * c * 512, ks), 1u);
        MMA_DONE();
        tl.eg_store(acc, 8 * c);
        ptx::wgmma_fence();
      }
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uyc + 4 * ks, mm.w_mn(um::IMG_WCL + 4 * 512, ks), ks > 0);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16_rs<1>(hacc, uyc + 4 * ks, mm.w_mn(um::IMG_WCL + 8 * 512, ks), ks > 0);
      mm.wgrad32(wIN, FG_E1, FG_FC3);
      MMA_DONE();
      TR_TILE(15);
      tl.eg_store(acc, EG_E2);
      tl.eg_store(hacc, EG_E2 + 8);
      __syncthreads();                                  // embedding-gradient tile: fragment layout -> point layout
      TR_TILE(16);
      // ---- PE backward: dproj_d = pi * sum_k 2^k g_{k,d} cos(pi 2^k proj_d), written as an fp16 block --------------
      {
        const float3 jt = tl.pe_backward<true>(tin);
        if constexpr (JOINT) {
          if (live) {
            float* o = jdt + (((size_t)b * R + ray) * S + sidx) * 6 + 3 * hsel;
            o[0] = jt.x; o[1] = jt.y; o[2] = jt.z;
          }
        }
      }
      TR_TILE(17);
      // dB += dproj^T [1 x y z ...]: the 21 real feature rows are in the first warpgroup's half; the second issues the
      // same instructions on rows that are never stored, which keeps the wgmma stream free of divergent branches
      OPERANDS_READY();
      mm.wgrad16(wDB, FG_DPR, FG_E1);
      MMA_DONE();
      __syncthreads();                                  // the next tile's PE overwrites E1 / E2 / DH
      TR_TILE(18);
      if constexpr (TRACE) ++tr_t;
    }
#undef OPERANDS_READY
#undef MMA_DONE
    }   // compute threads
    if constexpr (TRACE) tr_f0 = clock64();
    if (a.fwd_only) {                                   // nothing to reduce; the weight buffer is free once every warp is done
      __syncthreads();
      if (tid == 0 && gt < gt_end) {
        ptx::mbar_arrive_expect_tx(&misc->wbar, um::IMG_BYTES);
        ptx::bulk_g2s(smem + SM_W, image + (size_t)(gt / tpo) * um::IMG_BYTES, um::IMG_BYTES, &misc->wbar);
      }
      continue;
    }
    // ---- segment end: this CTA's partial sums for object b -----------------------------------------------------
    ls_d = warp_sum(ls_d); ls_c = warp_sum(ls_c); ls_o = warp_sum(ls_o);
    if (hsel == 0 && lane == 0) { float* l = misc->lsum[quad]; l[0] = ls_d; l[1] = ls_c; l[2] = ls_o; }
    __syncthreads();
    if (tid == 0 && gt < gt_end) {          // every MMA of this segment has completed: the weight buffer is free --
      ptx::mbar_arrive_expect_tx(&misc->wbar, um::IMG_BYTES);        // the next object's image lands during the flush
      ptx::bulk_g2s(smem + SM_W, image + (size_t)(gt / tpo) * um::IMG_BYTES, um::IMG_BYTES, &misc->wbar);
    }
    // the segment's gradient row is assembled in shared memory (the activation region is idle now: the scattered
    // 4-byte stores of the accumulator -> parameter-index mapping cost nothing there) and leaves as coalesced 16-byte stores
    float* Pr = reinterpret_cast<float*>(smem + SM_ACT0);
    if (tid < 3) {                                      // fixed summation order -> reproducible loss terms
      float s = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 4; ++w8) s += misc->lsum[w8][tid];
      Pr[L.P + tid] = s;
    }
    if (a.backward) {
      // accumulator fragments -> this segment's row of the partial block (plain stores, no atomics), then cleared for
      // the next object
      auto put = [&](float (&d)[16], int blk) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          int ld;
          const int base = wg_base(L, blk, fr0 + 8 * i, ld);
          if (base >= 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) Pr[base + (8 * j + 2 * cq + e) * ld] = d[4 * j + 2 * i + e] * INV_LS;
          }
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) d[k] = 0.f;
      };
      put(wIN, 0); put(wM1, 1); put(wCAT, 2); put(wM2, 3); put(wCL, 4);
      // heads tile: A = [fc4 | emb2 | hc], B = dhead (col 0 = alpha, 1..3 = colour); dB tile: A = dproj, B = emb1 cols [1, x, y, z]
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int ln = fr0 + 8 * i;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 2 * cq + e;
          const float vh = wHD[2 * i + e] * INV_LS, vb = wDB[2 * i + e] * INV_LS;
          if (col == 0) {
            if (ln < 32) Pr[L.o_Wa + ln] = vh;
            else if (ln == 32 + 42) Pr[L.o_ba] = vh;    // emb2's constant-1 column: the head biases
          } else if (col < 4) {
            if (ln == 32 + 42) Pr[L.o_boc + col - 1] = vh;
            else if (ln >= 80 && ln < 112) Pr[L.o_Woc + (col - 1) * 32 + (ln - 80)] = vh;
            if (ln < VMB_NDIRS) Pr[L.o_B + ln * 3 + col - 1] = vb;
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) { wHD[k] = 0.f; wDB[k] = 0.f; }
    }
    __syncthreads();
    {
      float4* dst = reinterpret_cast<float4*>(x.partials + (size_t)(blockIdx.x + b) * L.stride);
      const float4* src = reinterpret_cast<const float4*>(Pr);
      for (int i = tid; i < (L.stride >> 2); i += NT) dst[i] = src[i];
    }
    __syncthreads();
    if (tid == 0) {                                     // the row is out: one more of object b's segments is ready
      __threadfence();
      atomicAdd(&gbar[SY_OBJ + 2 * b], 1u);
    }
    if constexpr (TRACE) { tr_flush += clock64() - tr_f0; ++tr_nseg; }
  }
  TR_STAMP2(2, 9);
  if constexpr (TRACE) {
    if (tr_on) { tr[5] = (unsigned long long)tr_t; tr[6] = (unsigned long long)tr_flush; tr[7] = (unsigned long long)tr_nseg; }
  }

  if (!a.fwd_only) {
    // ---- finish: the reduction of every object's partial rows + AdamW, as a list of chunks (object, float4 column
    // range) in object order, handed out by a ticket counter to CTAs that have run all their tiles.  A chunk waits only
    // for ITS object's segments (ready count == segments), not for the whole grid: early objects are updated while
    // other CTAs still run tiles.  Each thread owns at most one float4 column of a chunk.
    const int n4 = L.stride >> 2;
    const int ncp = (n4 + NT - 1) / NT, csz = (n4 + ncp - 1) / ncp;   // chunks per object, columns per chunk
    const int nchunk = a.B * ncp;
    const bool upd = a.backward != 0;
    if (tid == 0) misc->ticket[0] = atomicAdd(&gbar[SY_TICKET], 1u);
    __syncthreads();
    TR_STAMP2(3, 10);
    for (int it = 0;; ++it) {
      const int k = (int)misc->ticket[it & 1];          // slot it & 1 was written before the last barrier
      if (k >= nchunk) break;
      const int b = k / ncp, i_lo = (k - b * ncp) * csz, i_hi = min(n4, i_lo + csz);
      const int c4 = i_lo + tid;
      const bool col = upd && c4 < i_hi, owner = i_lo == 0;
      const size_t row = (size_t)b * L.stride;
      // (1) everything that does not depend on other CTAs goes out before the wait: p / m / v (or grads) and the bias
      //     corrections of step t from the host-built table (torch's double-precision scalars, rounded once); beyond
      //     the table: 1 - beta^t = -expm1(t ln beta) in fp32 (cancellation-free, <= 3e-7 relative)
      float4 pp = make_float4(0.f, 0.f, 0.f, 0.f), mm = pp, vv = pp;
      if (col) {
        if (x.fuse_adam) {
          pp = *(reinterpret_cast<const float4*>(x.p + row) + c4);
          mm = *(reinterpret_cast<const float4*>(x.m + row) + c4);
          vv = *(reinterpret_cast<const float4*>(x.v + row) + c4);
        } else {
          pp = *(reinterpret_cast<const float4*>(a.grads + row) + c4);
        }
      }
      float step_size = x.step_size, bc2_sqrt = x.bc2_sqrt;
      if (x.fuse_adam && x.step_counter) {
        const int t = x.step_counter[b] + 1;
        if (t < x.bc_n) {
          const float2 bc = x.bc_table[t];
          step_size = (float)x.lr / bc.x;
          bc2_sqrt = bc.y;
        } else {
          step_size = (float)x.lr / (-expm1f((float)t * x.log_b1));
          bc2_sqrt = sqrtf(-expm1f((float)t * x.log_b2));
        }
      }
      const int c_first = cta_of_tile(rg, G, b * tpo), c_last = cta_of_tile(rg, G, (b + 1) * tpo - 1);
      const int nseg = c_last - c_first + 1;
      const float* P0 = x.partials + (size_t)(c_first + b) * L.stride;
      // (2) the next ticket, then wait until all of object b's segments have flushed their rows
      if (tid == 0) {
        misc->ticket[(it + 1) & 1] = atomicAdd(&gbar[SY_TICKET], 1u);
        long long w0 = 0;
        if constexpr (TRACE) w0 = clock64();
        const unsigned int* rdy = gbar + SY_OBJ + 2 * b;
        unsigned int spins = 0, r;
        for (;;) {
          asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(rdy) : "memory");
          if (r >= (unsigned int)nseg) break;
          __nanosleep(64);
          if (++spins > 400000000u) __trap();
        }
        if constexpr (TRACE) { tr_wait += clock64() - w0; ++tr_calls; }
      }
      __syncthreads();
      // (3) the object's loss terms and explosion guard (render_rays.py:88-90: the reference aborts before the
      //     update), and this column's rows, all loads in flight at once; both summed in segment order = CTA order,
      //     the same sums every run whichever CTA runs the chunk
      float l_d = 0.f, l_c = 0.f, l_o = 0.f;
      float4 gsum = make_float4(0.f, 0.f, 0.f, 0.f);
      const float4* src = reinterpret_cast<const float4*>(P0) + c4;
#pragma unroll 1
      for (int k0 = 0; k0 < nseg; k0 += 8) {
        float4 u[8];
        float lv[8][3];
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const bool in = k0 + kk < nseg;
          u[kk] = (in && col) ? __ldcg(src + (size_t)(k0 + kk) * n4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int j = 0; j < 3; ++j) lv[kk][j] = in ? __ldcg(P0 + (size_t)(k0 + kk) * L.stride + L.P + j) : 0.f;
        }
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          if (k0 + kk < nseg) {
            gsum.x += u[kk].x; gsum.y += u[kk].y; gsum.z += u[kk].z; gsum.w += u[kk].w;
            l_d += lv[kk][0]; l_c += lv[kk][1]; l_o += lv[kk][2];
          }
      }
      const float tot = l_d + a.cs * l_c + a.os * l_o;
      int bad = 0;
      if (x.guard_loss) {
        if (l_d > 100000.f || l_c > 100000.f || l_o > 100000.f) bad |= 1;
        if (!(tot == tot) || fabsf(tot) > 3.0e38f) bad |= 2;
      }
      if (owner && tid == 0) {
        float* lt = a.loss_terms + b * 4; lt[0] = l_d; lt[1] = l_c; lt[2] = l_o; lt[3] = tot;
        if (bad && x.status) atomicOr(x.status, bad);
        gbar[SY_OBJ + 2 * b + 1] = (unsigned int)bad;   // skip flag: the step number stays
      }
      // (4) update this thread's column: AdamW (fuse_adam; skipped for an exploded object) or grads += gradient
      if (col && !(bad && x.fuse_adam)) {
        const int e = c4 * 4;
        if (!x.fuse_adam) {
          float4 o = pp;
          o.x += gsum.x; o.y += gsum.y; o.z += gsum.z; o.w += gsum.w;
          if (e + 3 >= L.P) { if (e + 0 >= L.P) o.x = 0.f; if (e + 1 >= L.P) o.y = 0.f; if (e + 2 >= L.P) o.z = 0.f; o.w = 0.f; }
          *(reinterpret_cast<float4*>(a.grads + row) + c4) = o;
        } else {
          // torch.optim.AdamW._single_tensor_adamw, op for op as k_adamw restates it
          float* pj = &pp.x; float* mj = &mm.x; float* vj = &vv.x; const float* gj = &gsum.x;
          __half* img = x.image_out ? x.image_out + (size_t)b * x.img_halves : nullptr;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (e + j >= L.P) continue;
            float pw = pj[j] * x.lr_wd;
            const float m1 = mj[j] + (gj[j] - mj[j]) * x.one_m_b1;
            const float v1 = vj[j] * x.b2 + (x.one_m_b2 * gj[j]) * gj[j];
            const float denom = sqrtf(v1) / bc2_sqrt + x.eps;
            pw = pw - step_size * (m1 / denom);
            pj[j] = pw; mj[j] = m1; vj[j] = v1;
            if (img) {
              const int t = x.img_index[e + j];
              if (t >= 0) img[t] = __float2half_rn(pw);
              else if (t <= -2) reinterpret_cast<float*>(img)[-(t + 2)] = pw;
            }
          }
          *(reinterpret_cast<float4*>(x.p + row) + c4) = pp;
          *(reinterpret_cast<float4*>(x.m + row) + c4) = mm;
          *(reinterpret_cast<float4*>(x.v + row) + c4) = vv;
        }
      }
    }
    // ---- departure: the last CTA to leave has seen every chunk finish
    __threadfence();
    __syncthreads();
    if (tid == 0) misc->fin = (atomicAdd(&gbar[SY_DEPART], 1u) + 1u == (unsigned int)G) ? 1 : 0;
    __syncthreads();
    if (misc->fin) {                                    // the last CTA to leave: step numbers, re-arm the sync words
      __threadfence();
      if (x.fuse_adam && x.step_counter && a.backward)
        for (int b = tid; b < a.B; b += NT) if (gbar[SY_OBJ + 2 * b + 1] == 0u) x.step_counter[b] += 1;
      if (x.loss_sum && warp == 0) {                    // scalar loss of the step (loss.py:59-62), fixed summation order
        float s = 0.f;
        for (int b = lane; b < a.B; b += 32) s += __ldcg(a.loss_terms + b * 4 + 3);
        s = warp_sum(s);
        if (lane == 0) *x.loss_sum = s;
      }
      for (int b = tid; b < a.B; b += NT) gbar[SY_OBJ + 2 * b] = 0u;
      if (tid < SY_OBJ) gbar[tid] = 0u;
    }
  }
  TR_STAMP2(4, 11);
  if constexpr (TRACE) {
    if (tid == 0) { tr[12] = (unsigned long long)tr_wait; tr[13] = (unsigned long long)tr_calls; }
  }
#undef TR_STAMP
#undef TR_STAMP2
#undef TR_TILE
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static int fused_rows_needed(int n_obj, int n_sm) { return n_obj + n_sm; }

// Cost-aware split of B objects x tpo tiles over G CTAs, the CTAs with less work on the lowest object indices.
// Starting a second object inside a CTA costs it a flush of the gradient partial, a weight load and a pipeline refill,
// so tiles are laid out on a virtual axis x(t) = t + beta * (object of t) -- every object boundary is a gap of beta --
// and the axis is split from its end: CTA c, from the last down, takes the tiles that fit in ceil(rest / (c + 1)) of it,
// rest being the axis left for CTAs 0..c.  Rounding up puts the CTAs with one tile more on the last objects, so the
// first objects are complete, and their finish chunks run, while those CTAs run their last tile.  beta is the largest
// of {1, 0.7, 0.4, 0} whose split keeps every CTA at the fewest tiles possible, ceil(tiles / G).
static void fused_partition(int B, int tpo, int G, uf::Ranges& rg) {
  const long long T = (long long)B * tpo;
  const long long rounds = (T + G - 1) / G;
  for (double beta : {1.0, 0.7, 0.4, 0.0}) {
    if (beta > 0.0 && T < 2LL * G) continue;
    auto x = [&](long long t) { return (double)t + beta * (double)(t / tpo); };
    rg.begin[G] = (int)T;
    long long most = 0;
    for (int c = G - 1; c > 0; --c) {                   // G <= T: every CTA keeps at least one tile
      const long long end = rg.begin[c + 1];
      const double top = x(end - 1) + 1.0, cap = std::ceil(top / (c + 1) - 1e-9);
      long long p = end - 1;
      while (p - 1 >= c && top - x(p - 1) <= cap) --p;
      rg.begin[c] = (int)p;
      most = std::max(most, end - p);
    }
    rg.begin[0] = 0;
    most = std::max(most, (long long)rg.begin[1]);
    if (most <= rounds) return;
  }
}

// jdt: the joint step's [B][R * S][2][3] pose-gradient halves (JOINT instantiations), or nullptr (the plain step).
// trace: [2 * grid][uf::TR_STRIDE] phase stamps (the TRACE instantiation, training step at S = 10 only), or nullptr
static int fused_launch_step(const VmbLayout& L, const StepParams& sp, const FusedExtra& fx, const void* image, int n_sm,
                             cudaStream_t st, std::string& err, float* jdt = nullptr, unsigned long long* trace = nullptr) {
  using namespace uf;
  if (L.H != 32 || L.nfreq != 6) { err = "fused step kernel: hidden must be 32 and n_freq 6"; return VMB_E_UNSUPPORTED; }
  if (sp.S < 1 || sp.S > 32) { err = "fused step kernel: n_samples must be in [1, 32]"; return VMB_E_UNSUPPORTED; }
  if (!sp.fwd_only && sp.B > MAX_OBJ_SMEM) {
    err = "fused step kernel: too many objects for the in-kernel mask counts"; return VMB_E_UNSUPPORTED;
  }
  if (jdt && (sp.fwd_only || !sp.backward)) { err = "fused step kernel: the joint step needs the backward"; return VMB_E_UNSUPPORTED; }
  if (trace && (jdt || sp.fwd_only || !sp.backward || sp.S != 10)) {
    err = "fused step kernel: the phase trace covers the training step at n_samples 10 only"; return VMB_E_UNSUPPORTED;
  }
  int dev = 0;
  cudaGetDevice(&dev);
  const int smem_bytes = SM_CNT + (sp.fwd_only ? 0 : sp.B * 12) + SMEM_SLACK;
  {
    cudaError_t e = cudaSuccess;
    for (auto raise : {smem_limit_once<k_step_fused<0, false>>, smem_limit_once<k_step_fused<10, false>>,
                       smem_limit_once<k_step_fused<14, false>>, smem_limit_once<k_step_fused<0, true>>,
                       smem_limit_once<k_step_fused<10, true>>, smem_limit_once<k_step_fused<14, true>>,
                       smem_limit_once<k_step_fused<10, false, true>>})
      if (e == cudaSuccess) e = raise(dev, SMEM_MAX);
    if (e != cudaSuccess) { err = std::string("cudaFuncSetAttribute(k_step_fused): ") + cudaGetErrorString(e); return VMB_E_CUDA; }
  }
  const int rpw = 32 / sp.S;                  // whole rays per warp: the sample axis never crosses a warp
  const int nr = 4 * rpw;
  const int tpo = (sp.R + nr - 1) / nr;       // tiles per object
  const long long T = (long long)tpo * sp.B;
  if (T > 0x7fffffffLL) { err = "fused step kernel: too many tiles"; return VMB_E_ARG; }
  long long grid = T;
  if (grid > n_sm) grid = n_sm;
  if (grid > MAX_CTAS) grid = MAX_CTAS;
  if (grid < 1) grid = 1;
  Ranges rg;
  fused_partition(sp.B, tpo, (int)grid, rg);
  const unsigned char* img = (const unsigned char*)image;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(NT); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  // a training launch's finish waits on other CTAs' segments: every CTA must be resident (grid <= #SMs, one CTA per
  // SM), and the cooperative attribute makes the runtime guarantee it
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = sp.fwd_only ? 0 : 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaError_t e;
  auto kern = [&](auto k) { return cudaLaunchKernelEx(&cfg, k, sp, fx, L, img, rg, tpo, nr, rpw, jdt, trace); };
  if (trace) e = kern(k_step_fused<10, false, true>);
  else if (jdt) e = kern(sp.S == 10 ? k_step_fused<10, true> : sp.S == 14 ? k_step_fused<14, true> : k_step_fused<0, true>);
  else     e = kern(sp.S == 10 ? k_step_fused<10, false> : sp.S == 14 ? k_step_fused<14, false> : k_step_fused<0, false>);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { err = std::string("k_step_fused launch: ") + cudaGetErrorString(e); return VMB_E_CUDA; }
  return 0;
}
