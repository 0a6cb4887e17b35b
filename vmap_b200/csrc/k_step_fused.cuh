// K1: ONE launch per optimisation step for hidden = 32 (sm_90a: wgmma, bulk async copy, mbarrier).
//   mask counts (render_rays.py:68,86) -> PE -> MLP -> volume render -> losses -> backward
//   -> per-object gradient reduction in a fixed order -> AdamW + fp16 weight-image refresh
// fp16 operands / fp32 accumulate on wgmma.mma_async (m64nNk16, both operands from shared memory, accumulators in
// registers), weights staged per object with one bulk async copy.  CTA = 256 threads = two warpgroups; a tile is up to
// 128 sample points (whole rays) and walks through 12 dependent MMA stages (6 forward, 6 backward): threads write the
// stage's operands -> fence + CTA barrier -> each warpgroup issues the stage's wgmmas for its 64 points and waits ->
// the hidden-layer epilogues run on the accumulator fragments in registers.  Shared-memory operand layout: no-swizzle
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
//   * K0 (mask counts) runs in the prologue, K2 (AdamW) in the last CTA to finish an object: every (CTA, object)
//     segment writes its gradient partial to its own row, the finisher adds the rows in segment order (bitwise
//     reproducible -- no floating-point atomics anywhere) and applies AdamW exactly as k_adamw does.
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
  unsigned int* obj_done;     // [B] segments finished per object (non-cooperative), [B] skip flags, [2] grid arrive / depart (self-resetting)
  const int* counts_in;       // optional [B][4] external mask counts (ray-sharded iMAP: all-reduced by the caller)
  int* counts_pub;            // [B][4] scratch: cooperative launches count each object ONCE (CTA b mod grid) and publish here
  int fuse_adam;              // 1: the finisher applies AdamW; 0: it adds the reduced gradient into `grads`
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
  int cooperative;            // 1: cooperative launch (all CTAs resident): an object's CTAs share its reduction + update
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
constexpr int MAX_OBJ_SMEM = (SMEM_MAX - SM_CNT) / 12;            // objects whose counts fit
constexpr float LS = um::LS, INV_LS = um::INV_LS;

struct Misc {
  uint64_t wbar;
  int on[3];
  int fin, skip;
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

// Work partition: CTA c owns tile pairs [begin[c], begin[c+1]) of the global list (object-major).  Built on the host
// (fused_partition) so that a CTA whose range crosses an object boundary -- it pays a second flush / weight load /
// pipeline fill -- gets correspondingly fewer pairs: no CTA's cost exceeds the even share by more than one pair.
constexpr int MAX_CTAS = 192;
struct Ranges { int begin[MAX_CTAS + 1]; };
__device__ __forceinline__ int cta_of_pair(const Ranges& rg, int G, int pair) {        // largest c with begin[c] <= pair
  int lo = 0, hi = G - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (rg.begin[mid] <= pair) lo = mid; else hi = mid - 1; }
  return lo;
}

}  // namespace uf

// ---------------------------------------------------------------------------------------------------------------
template <int SC>
__global__ void __launch_bounds__(uf::NT, 1)
k_step_fused(StepParams a, FusedExtra x, VmbLayout L, const unsigned char* image, const __grid_constant__ uf::Ranges rg, int tpo, int npo, int nr, int rpw) {
  using namespace uf;
  extern __shared__ __align__(1024) unsigned char smem[];
  Misc* misc = reinterpret_cast<Misc*>(smem + SM_MISC);
  int* cnt = reinterpret_cast<int*>(smem + SM_CNT);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S = SC ? SC : a.S, R = a.R;

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
    ptx::bulk_g2s(smem + SM_W, image + (size_t)(gt_begin / npo) * um::IMG_BYTES, um::IMG_BYTES, &misc->wbar);
  }
  // ---- K0 in the prologue: mask counts of EVERY object (the any-empty early-out couples them, render_rays.py:68-73).
  // Cooperative launch: CTA c counts objects c, c + grid, ... ONCE and publishes counts + empty flags + a "published"
  // counter in global memory; every CTA starts its tiles at once and acquires the counts right before its first
  // volume render (thousands of cycles later: the wait is free).  Otherwise every CTA counts everything (every CTA
  // reads all the label / mask bytes).
  const bool pub_counts = x.cooperative && !x.counts_in && !a.fwd_only;
  unsigned int* gbar = x.obj_done + 2 * a.B;            // [0] arrive, [1] depart, [2] objects published, [3..5] empty flags
  if (pub_counts) {
    for (int b = blockIdx.x; b < a.B; b += G) {
      if (tid < 3) cnt[tid] = 0;
      __syncthreads();
      const unsigned char* s = a.sem + (size_t)b * a.sem_stride;
      const unsigned char* m = a.mask + (size_t)b * a.mask_stride;
      const bool vec = (((size_t)s | (size_t)m) & 3) == 0;
      const int nw = vec ? (R >> 2) : 0;
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
          if (cnt[k] == 0) atomicOr(&gbar[3 + k], 1u);
        }
        __threadfence();
        atomicAdd(&gbar[2], 1u);
      }
      __syncthreads();
    }
  } else if (!a.fwd_only) {
    if (x.counts_in) {
      for (int i = tid; i < a.B * 3; i += NT) {
        const int c = x.counts_in[(i / 3) * 4 + (i % 3)];
        cnt[i] = c;
        if (c == 0) misc->on[i % 3] = 0;
      }
    } else {
      // warp w counts objects w, w + NT/32, ...; two objects at a time with every load of both in flight together (the
      // inputs are cold in HBM: one latency per pair of objects instead of one per 8 words)
      const int nw = R >> 2;
      auto finish = [&](int b, int nd, int no, int ns) {
        const unsigned char* s = a.sem + (size_t)b * a.sem_stride;
        const unsigned char* m = a.mask + (size_t)b * a.mask_stride;
        const bool vec = (((size_t)s | (size_t)m) & 3) == 0;
        for (int r = (vec ? (nw << 2) : 0) + lane; r < R; r += 32) {      // tail rays, or everything when unaligned
          const int sv = s[r], mo = sv != 0;
          nd += (m[r] != 0) & mo; no += mo; ns += sv != 2;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          nd += __shfl_xor_sync(0xffffffffu, nd, o); no += __shfl_xor_sync(0xffffffffu, no, o); ns += __shfl_xor_sync(0xffffffffu, ns, o);
        }
        if (lane == 0) {
          cnt[b * 3] = nd; cnt[b * 3 + 1] = no; cnt[b * 3 + 2] = ns;
          if (nd == 0) misc->on[0] = 0;
          if (no == 0) misc->on[1] = 0;
          if (ns == 0) misc->on[2] = 0;
        }
      };
      // every CTA needs every object's counts: each starts at a different object, so the grid does not hit the same
      // cache lines at the same moment
      const int shift = (int)((blockIdx.x * 7u) % (unsigned)a.B);
      for (int iA = warp; iA < a.B; iA += 2 * (NT / 32)) {
        const int iB = iA + NT / 32;
        const bool hasB = iB < a.B;
        const int bA = (iA + shift) % a.B, bB = hasB ? (iB + shift) % a.B : bA;
        const uint32_t* sA = reinterpret_cast<const uint32_t*>(a.sem + (size_t)bA * a.sem_stride);
        const uint32_t* mA = reinterpret_cast<const uint32_t*>(a.mask + (size_t)bA * a.mask_stride);
        const uint32_t* sB = reinterpret_cast<const uint32_t*>(a.sem + (size_t)(hasB ? bB : bA) * a.sem_stride);
        const uint32_t* mB = reinterpret_cast<const uint32_t*>(a.mask + (size_t)(hasB ? bB : bA) * a.mask_stride);
        const bool vA = (((size_t)sA | (size_t)mA) & 3) == 0, vB = hasB && (((size_t)sB | (size_t)mB) & 3) == 0;
        int cA[3] = {0, 0, 0}, cB[3] = {0, 0, 0};
        for (int w0 = 0; w0 < nw; w0 += 320) {                  // four rays per 32-bit load, ten loads per array per lane
          uint32_t sa[10], ma[10], sb[10], mb[10];
#pragma unroll
          for (int u = 0; u < 10; ++u) {
            const int w = w0 + u * 32 + lane;
            const bool in = w < nw;
            sa[u] = (in && vA) ? __ldg(sA + w) : 0u;  ma[u] = (in && vA) ? __ldg(mA + w) : 0u;
            sb[u] = (in && vB) ? __ldg(sB + w) : 0u;  mb[u] = (in && vB) ? __ldg(mB + w) : 0u;
          }
          // one bit per byte: nonzero(x) folds a byte's bits into bit 0 (labels are 0 / 1 / 2, masks any nonzero = true)
          auto nzb = [](uint32_t v) { v |= v >> 4; v |= v >> 2; v |= v >> 1; return v & 0x01010101u; };
#pragma unroll
          for (int u = 0; u < 10; ++u) {
            const bool in = w0 + u * 32 + lane < nw;
            const uint32_t oa = (in && vA) ? nzb(sa[u]) : 0u, ob = (in && vB) ? nzb(sb[u]) : 0u;
            cA[1] += __popc(oa); cA[0] += __popc(oa & nzb(ma[u])); cA[2] += (in && vA) ? __popc(nzb(sa[u] ^ 0x02020202u)) : 0;
            cB[1] += __popc(ob); cB[0] += __popc(ob & nzb(mb[u])); cB[2] += (in && vB) ? __popc(nzb(sb[u] ^ 0x02020202u)) : 0;
          }
        }
        finish(bA, cA[0], cA[1], cA[2]);
        if (hasB) finish(bB, cB[0], cB[1], cB[2]);
      }
    }
  }
  __syncthreads();

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
  const float* Bd = wf + um::F_DIRS;
  // ... and accumulator-fragment layout (wgmma m64nN): this thread holds rows fr0 and fr0 + 8, columns 8j + 2 cq + {0, 1}
  const int cq = lane & 3, fr0 = 64 * hsel + 16 * quad + (lane >> 2);
  Mma mm;
  mm.a16 = ptx::smem_u32(act) >> 4;
  mm.w16 = ptx::smem_u32(smem + SM_W) >> 4;
  mm.mh = hsel;
  // persistent weight-gradient accumulators of the current object (this warpgroup's 64 feature rows)
  float wIN[16] = {}, wM1[16] = {}, wCAT[16] = {}, wM2[16] = {}, wCL[16] = {}, wHD[8] = {}, wDB[8] = {};
  // loss weights of this thread's current object: (term enabled: no object has an empty mask) / (this object's mask count)
  const float on_d = misc->on[0] ? 1.f : 0.f, on_c = misc->on[1] ? 1.f : 0.f, on_o = misc->on[2] ? 1.f : 0.f;
  float w_d = 0.f, w_c = 0.f, w_o = 0.f;
  bool cnt_ready = !pub_counts;       // published counts acquired?

  // Reduce object b's partial rows over float4 columns [i_lo, i_hi) in segment order (the same sum every run) and either
  // apply AdamW (fuse_adam) or add the reduced gradient into `grads`.  `owner` writes the object's loss terms / status.
  // Called by all threads of the CTA; returns the object's skip flag (loss explosion guard, render_rays.py:88-90).
  auto finish_rows = [&](int b, int i_lo, int i_hi, bool owner) -> int {
    const int c_first = cta_of_pair(rg, G, b * npo), c_last = cta_of_pair(rg, G, (b + 1) * npo - 1);
    const int nseg = c_last - c_first + 1;
    const float* P0 = x.partials + (size_t)(c_first + b) * L.stride;
    const size_t row = (size_t)b * L.stride;
    const int n4 = L.stride >> 2;
    const bool upd = a.backward != 0;
    // (1) the object's loss terms (segment order), the explosion guard and the bias corrections
    if (warp == 0) {
      float s = 0.f;
      if (nseg <= 10) {                                 // up to ten segments are loaded by 30 lanes at once
        const int k = lane / 3, j = lane - 3 * k;
        const float v = (k < nseg) ? __ldcg(P0 + (size_t)k * L.stride + L.P + j) : 0.f;
        for (int kk = 0; kk < nseg; ++kk) s += __shfl_sync(0xffffffffu, v, kk * 3 + (lane < 3 ? lane : 0));
      } else if (lane < 3) {
        for (int k = 0; k < nseg; ++k) s += __ldcg(P0 + (size_t)k * L.stride + L.P + lane);
      }
      const float l_d = __shfl_sync(0xffffffffu, s, 0), l_c = __shfl_sync(0xffffffffu, s, 1), l_o = __shfl_sync(0xffffffffu, s, 2);
      if (lane == 0) {
        const float tot = l_d + a.cs * l_c + a.os * l_o;
        if (owner) { float* lt = a.loss_terms + b * 4; lt[0] = l_d; lt[1] = l_c; lt[2] = l_o; lt[3] = tot; }
        int bad = 0;                                    // render_rays.py:88-90: the reference aborts before the update
        if (x.guard_loss) {
          if (l_d > 100000.f || l_c > 100000.f || l_o > 100000.f) bad |= 1;
          if (!(tot == tot) || fabsf(tot) > 3.0e38f) bad |= 2;
          if (bad && x.status && owner) atomicOr(x.status, bad);
        }
        misc->skip = bad;
        if (x.fuse_adam && x.step_counter) {
          // bias corrections of step t from the host-built table (torch's double-precision scalars, rounded once);
          // beyond the table: 1 - beta^t = -expm1(t ln beta) in fp32 (cancellation-free, <= 3e-7 relative)
          const int t = x.step_counter[b] + 1;
          if (t < x.bc_n) {
            const float2 bc = x.bc_table[t];
            misc->step_size = (float)x.lr / bc.x;
            misc->bc2_sqrt = bc.y;
          } else {
            misc->step_size = (float)x.lr / (-expm1f((float)t * x.log_b1));
            misc->bc2_sqrt = sqrtf(-expm1f((float)t * x.log_b2));
          }
        } else {
          misc->step_size = x.step_size; misc->bc2_sqrt = x.bc2_sqrt;
        }
      }
    }
    __syncthreads();
    const int sk = misc->skip;
    // (2) reduce + update this CTA's columns (normally at most one float4 column per thread).  Deliberately compact
    //     code: it runs once per launch out of a cold instruction cache, where instruction fetch, not data, is the cost
    if (upd && !(sk && x.fuse_adam)) {
      const float step_size = misc->step_size, bc2_sqrt = misc->bc2_sqrt;
      for (int c4 = i_lo + tid; c4 < i_hi; c4 += NT) {
        const float4* src = reinterpret_cast<const float4*>(P0) + c4;
        float4 pp, mm = make_float4(0.f, 0.f, 0.f, 0.f), vv = mm;
        if (x.fuse_adam) {
          pp = *(reinterpret_cast<const float4*>(x.p + row) + c4);
          mm = *(reinterpret_cast<const float4*>(x.m + row) + c4);
          vv = *(reinterpret_cast<const float4*>(x.v + row) + c4);
        } else {
          pp = *(reinterpret_cast<const float4*>(a.grads + row) + c4);
        }
        // segment order = CTA order: the same sum every run; four rows in flight per batch
        float4 gsum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
        for (int k0 = 0; k0 < nseg; k0 += 4) {
          float4 u[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) u[k] = (k0 + k < nseg) ? __ldcg(src + (size_t)(k0 + k) * n4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k0 + k < nseg) { gsum.x += u[k].x; gsum.y += u[k].y; gsum.z += u[k].z; gsum.w += u[k].w; }
        }
        const int e = c4 * 4;
        if (!x.fuse_adam) {
          float4 o = pp;
          o.x += gsum.x; o.y += gsum.y; o.z += gsum.z; o.w += gsum.w;
          if (e + 3 >= L.P) { if (e + 0 >= L.P) o.x = 0.f; if (e + 1 >= L.P) o.y = 0.f; if (e + 2 >= L.P) o.z = 0.f; o.w = 0.f; }
          *(reinterpret_cast<float4*>(a.grads + row) + c4) = o;
          continue;
        }
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
    __syncthreads();                                    // the next call's warp 0 overwrites misc->skip
    return sk;
  };

  // The work list is in units of TILE PAIRS (two consecutive tiles of an object, run one after the other), which is
  // the unit the host-side partition balances.
  for (long long gt = gt_begin; gt < gt_end;) {
    const int b = (int)(gt / npo);
    const int p0 = (int)(gt - (long long)b * npo);
    const int p1 = (int)min((long long)npo, (long long)p0 + (gt_end - gt));
    gt += p1 - p0;
    const int t0 = 2 * p0, t1 = min(2 * p1, tpo);       // this segment's tiles of object b

    // ---- this object's weight image (one bulk copy global -> shared, issued before the previous segment's flush) ----
    um::mbar_wait_or_trap(&misc->wbar, wpar);
    wpar ^= 1;

    float ls_d = 0.f, ls_c = 0.f, ls_o = 0.f;
    {
    const float isc = 1.0f / a.scale[b];
    bool seg_w = false;               // w_d / w_c / w_o hold this segment's object?
    if (!a.fwd_only && !pub_counts) {
      w_d = on_d / ((float)cnt[b * 3 + 0] + 1e-10f);
      w_c = on_c / ((float)cnt[b * 3 + 1] + 1e-10f);
      w_o = on_o / ((float)cnt[b * 3 + 2] + 1e-10f);
      seg_w = true;
    }

    // A stage: operands written by generic stores -> fence for the async proxy -> CTA barrier -> each warpgroup issues
    // the stage's wgmmas on its M half and, behind them, the layer's weight-gradient wgmmas into the persistent
    // accumulators -> commit -> wait.
#define OPERANDS_READY() do { ptx::fence_async_smem(); __syncthreads(); ptx::wgmma_fence(); } while (0)
#define MMA_DONE() do { ptx::wgmma_commit(); ptx::wgmma_wait<0>(); } while (0)
    // hidden-layer epilogue on the fragment: acc + bias -> ReLU -> fp16 into block FG
    auto epi_relu = [&](const float (&v)[16], int bias_off, int fg) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 bb = *reinterpret_cast<const float2*>(wf + bias_off + 8 * j + 2 * cq);
        unsigned char* dst = act + (fg + j) * FGB + fr0 * 16 + cq * 4;
        *reinterpret_cast<uint32_t*>(dst) = pack_relu_h2(v[4 * j] + bb.x, v[4 * j + 1] + bb.y);
        *reinterpret_cast<uint32_t*>(dst + 128) = pack_relu_h2(v[4 * j + 2] + bb.x, v[4 * j + 3] + bb.y);
      }
    };
    // dgrad epilogue: dY = (h > 0) * acc; h is read from its own block, dY goes to a block whose readers retired
    auto epi_dgrad = [&](const float (&v)[16], int fg_h, int fg_out) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int off = j * FGB + fr0 * 16 + cq * 4;
        const uint32_t h0 = *reinterpret_cast<const uint32_t*>(act + fg_h * FGB + off);
        const uint32_t h1 = *reinterpret_cast<const uint32_t*>(act + fg_h * FGB + off + 128);
        *reinterpret_cast<uint32_t*>(act + fg_out * FGB + off) = um::gate_h2(um::pack_h2(v[4 * j], v[4 * j + 1]), h0);
        *reinterpret_cast<uint32_t*>(act + fg_out * FGB + off + 128) = um::gate_h2(um::pack_h2(v[4 * j + 2], v[4 * j + 3]), h1);
      }
    };
    // embedding-gradient fragment (8-column groups starting at 4-column block blk0) -> the shared fp32 tile
    auto eg_store = [&](const auto& v, int blk0) {
      constexpr int NJ = (int)(sizeof(v) / 16);
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        float* d = reinterpret_cast<float*>(eg + (blk0 + 2 * j + (cq >> 1)) * FGB + fr0 * 16 + (cq & 1) * 8);
        *reinterpret_cast<float2*>(d) = make_float2(v[4 * j], v[4 * j + 1]);
        *reinterpret_cast<float2*>(d + 32) = make_float2(v[4 * j + 2], v[4 * j + 3]);
      }
    };
    // eight consecutive embedding-gradient columns of this thread's point
    auto eg_load8 = [&](int blk, float (&o)[8]) {
      const float4 u0 = *reinterpret_cast<const float4*>(eg + blk * FGB + p * 16);
      const float4 u1 = *reinterpret_cast<const float4*>(eg + (blk + 1) * FGB + p * 16);
      o[0] = u0.x; o[1] = u0.y; o[2] = u0.z; o[3] = u0.w; o[4] = u1.x; o[5] = u1.y; o[6] = u1.z; o[7] = u1.w;
    };

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
      const int ray = t * nr + ray_in_tile;
      // ---- E0: positional embedding (embedding.py:82-91) ----------------------------------------------------
      const float t0x = nx * isc, t1x = ny * isc, t2x = nz * isc, zv = nzv;
      const uint64_t tp0 = um::pk2(t0x, t0x), tp1 = um::pk2(t1x, t1x), tp2 = um::pk2(t2x, t2x);
      const float gd = n_gd, gc0 = n_c0, gc1 = n_c1, gc2 = n_c2;
      const int sv = n_sem, mv = n_msk;
      const bool live = n_live;
      prefetch(t + 1);
      {
        uint4* e1 = reinterpret_cast<uint4*>(act + FG_E1 * FGB + p * 16);
        uint4* e2 = reinterpret_cast<uint4*>(act + FG_E2 * FGB + p * 16);
        const int q0 = hsel ? 3 : 0, q1 = hsel ? 5 : 3;
        // software pipeline over the 4-direction chunks: the NEXT chunk's projections, range reduction and MUFU
        // sin / cos are issued before the CURRENT chunk's doubling recurrence, which hides their latency
        uint64_t s01, s23, c01, c23;
        {
          uint64_t pj01, pj23;
          um::project4(Bd, q0, tp0, tp1, tp2, pj01, pj23);
          um::sincos4_x2(pj01, pj23, s01, s23, c01, c23);
        }
#pragma unroll 1
        for (int q = q0; q < q1; ++q) {                // directions 4q .. 4q+3
          float sv[4][6];
          uint64_t ns01 = 0, ns23 = 0, nc01 = 0, nc23 = 0;
          if (q + 1 < q1) {
            uint64_t pj01, pj23;
            um::project4(Bd, q + 1, tp0, tp1, tp2, pj01, pj23);
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
          um::sin_ladder(fmaf(Bd[2 * um::DIRS_PITCH + 20], t2x, fmaf(Bd[um::DIRS_PITCH + 20], t1x, Bd[20] * t0x)), s);
          const uint4 u0 = make_uint4(um::pack_h2(1.0f, t0x), um::pack_h2(t1x, t2x), um::pack_h2(s[0], s[1]), um::pack_h2(s[2], s[3]));
          const uint4 u5 = make_uint4(um::pack_h2(s[4], s[5]), um::pack_h2(1.0f, 0.f), 0u, 0u);
          e1[0] = u0;
          e2[5 * 128] = u5;
          e1[11 * 128] = make_uint4(0u, 0u, 0u, 0u);
          // zero this point's dhead row (cols 4..15 stay zero; 0..3 are written after the render)
          uint4* dh = reinterpret_cast<uint4*>(act + FG_DH * FGB + p * 16);
          dh[0] = make_uint4(0u, 0u, 0u, 0u); dh[128] = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      float acc[16], hacc[8];
      OPERANDS_READY();                                 // in_layer: emb1 (K = 96)
#pragma unroll
      for (int ks = 0; ks < 6; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_E1, ks), mm.w_k(um::IMG_WIN, ks), ks > 0);
      MMA_DONE();
      epi_relu(acc, um::F_BIN, FG_FC1);
      OPERANDS_READY();                                 // mid1: fc1
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_FC1, ks), mm.w_k(um::IMG_WM1, ks), ks > 0);
      MMA_DONE();
      epi_relu(acc, um::F_BM1, FG_FC2);
      OPERANDS_READY();                                 // cat_layer: [fc2 | emb1] (K = 128)
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_FC2, ks), mm.w_k(um::IMG_WCAT, ks), ks > 0);
      MMA_DONE();
      epi_relu(acc, um::F_BCAT, FG_FC3);
      OPERANDS_READY();                                 // mid2: fc3
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_FC3, ks), mm.w_k(um::IMG_WM2, ks), ks > 0);
      MMA_DONE();
      epi_relu(acc, um::F_BM2, FG_FC4);
      OPERANDS_READY();                                 // color_linear: [fc4 | emb2] (K = 80) ; out_alpha: fc4 -> column 0
#pragma unroll
      for (int ks = 0; ks < 5; ++ks) ptx::wgmma_n32<0, 0>(acc, mm.a_k(FG_FC4, ks), mm.w_k(um::IMG_WCL, ks), ks > 0);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16<0, 0>(hacc, mm.a_k(FG_FC4, ks), mm.w16_k(um::IMG_WA16, ks), ks > 0);
      MMA_DONE();
      epi_relu(acc, um::F_BCL, FG_HC);
      if (cq == 0) { hd[fr0 * 4] = hacc[0]; hd[(fr0 + 8) * 4] = hacc[2]; }
      OPERANDS_READY();                                 // out_color: hc -> columns 1..3
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16<0, 0>(hacc, mm.a_k(FG_HC, ks), mm.w16_k(um::IMG_WOC16, ks), ks > 0);
      MMA_DONE();
      if (cq == 0) { hd[fr0 * 4 + 1] = hacc[1]; hd[(fr0 + 8) * 4 + 1] = hacc[3]; }
      if (cq == 1) { hd[fr0 * 4 + 2] = hacc[0]; hd[fr0 * 4 + 3] = hacc[1]; hd[(fr0 + 8) * 4 + 2] = hacc[2]; hd[(fr0 + 8) * 4 + 3] = hacc[3]; }
      __syncthreads();                                  // heads tile: fragment layout -> point layout
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
        if (!seg_w && pub_counts) {                     // cooperative launch: acquire the published mask counts (first render only)
          if (!cnt_ready) {
            const volatile unsigned int* pubd = gbar + 2;
            unsigned int spins = 0;
            while (*pubd < (unsigned int)a.B) { if (++spins > 2000000000u) __trap(); }
            __threadfence();
            cnt_ready = true;
          }
          const volatile unsigned int* ef = gbar + 3;
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
      if (a.fwd_only || !a.backward) { __syncthreads(); continue; }
      OPERANDS_READY();                                 // d_hc = dhead @ W_oc ; heads wgrad (out_alpha + out_color, weights and biases)
      ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_DH, 0), mm.w16_mn(um::IMG_WOC16), 0u);
      mm.wgrad16(wHD, FG_FC4, FG_DH);
      MMA_DONE();
      epi_dgrad(acc, FG_HC, FG_Z);                      // dYc -> Z
      OPERANDS_READY();                                 // d_fc4 = dYc @ W_cl[:, :32] + dhead @ W_a ; wgrad color_linear
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_Z, ks), mm.w_mn(um::IMG_WCL, ks), ks > 0);
      ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_DH, 0), mm.w16_mn(um::IMG_WA16), 1u);
      mm.wgrad32(wCL, FG_FC4, FG_Z);
      MMA_DONE();
      epi_dgrad(acc, FG_FC4, FG_HC);                    // dY4 -> HC
      OPERANDS_READY();                                 // d_fc3 = dY4 @ W_m2 ; wgrad mid2
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_HC, ks), mm.w_mn(um::IMG_WM2, ks), ks > 0);
      mm.wgrad32(wM2, FG_FC3, FG_HC);
      MMA_DONE();
      epi_dgrad(acc, FG_FC3, FG_FC4);                   // dY3 -> FC4
      OPERANDS_READY();                                 // d_fc2 = dY3 @ W_cat[:, :32] ; wgrad cat_layer
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_FC4, ks), mm.w_mn(um::IMG_WCAT, ks), ks > 0);
      mm.wgrad32(wCAT, FG_FC2, FG_FC4);
      MMA_DONE();
      epi_dgrad(acc, FG_FC2, FG_HC);                    // dY2 -> HC
      OPERANDS_READY();                                 // d_fc1 = dY2 @ W_m1 ; wgrad mid1
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_HC, ks), mm.w_mn(um::IMG_WM1, ks), ks > 0);
      mm.wgrad32(wM1, FG_FC1, FG_HC);
      MMA_DONE();
      epi_dgrad(acc, FG_FC1, FG_FC3);                   // dY1 -> FC3
      // d_emb1 = dY3 @ W_cat[:, 32:] + dY1 @ W_in (32 columns at a time), d_emb2 = dYc @ W_cl[:, 32:] ; wgrad in_layer
      OPERANDS_READY();
#pragma unroll
      for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_FC4, ks), mm.w_mn(um::IMG_WCAT + (4 + 4 * c) * 512, ks), ks > 0);
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_FC3, ks), mm.w_mn(um::IMG_WIN + 4 * c * 512, ks), 1u);
        MMA_DONE();
        eg_store(acc, 8 * c);
        ptx::wgmma_fence();
      }
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32<0, 1>(acc, mm.a_k(FG_Z, ks), mm.w_mn(um::IMG_WCL + 4 * 512, ks), ks > 0);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16<0, 1>(hacc, mm.a_k(FG_Z, ks), mm.w_mn(um::IMG_WCL + 8 * 512, ks), ks > 0);
      mm.wgrad32(wIN, FG_E1, FG_FC3);
      MMA_DONE();
      eg_store(acc, EG_E2);
      eg_store(hacc, EG_E2 + 8);
      __syncthreads();                                  // embedding-gradient tile: fragment layout -> point layout
      // ---- PE backward: dproj_d = pi * sum_k 2^k g_{k,d} cos(pi 2^k proj_d), written as an fp16 block --------------
      {
        const int q0 = hsel ? 3 : 0, q1 = hsel ? 5 : 3;
        uint64_t c01, c23;
        {
          uint64_t pj01, pj23;
          um::project4(Bd, q0, tp0, tp1, tp2, pj01, pj23);
          um::cos4_x2(pj01, pj23, c01, c23);
        }
#pragma unroll 1
        for (int q = q0; q < q1; ++q) {
          float g1a[8], g1b[8], g2[8];
          eg_load8(4 * q + 2, g1a);                    // emb1 cols of directions 4q, 4q+1 (k = 0..3)
          eg_load8(4 * q + 4, g1b);                    //                          4q+2, 4q+3
          eg_load8(EG_E2 + 2 * q, g2);                 // emb2 cols (k = 4, 5)
          float cv[4][6], dp[4];
          uint64_t nc01 = 0, nc23 = 0;
          if (q + 1 < q1) {                            // next chunk's front half before this chunk's recurrence
            uint64_t pj01, pj23;
            um::project4(Bd, q + 1, tp0, tp1, tp2, pj01, pj23);
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
          }
          // directions 4q..4q+3 = columns (4q)%8.. of feature group q/2
          *reinterpret_cast<uint2*>(act + (FG_DPR + (q >> 1)) * FGB + p * 16 + (q & 1) * 8) =
              make_uint2(um::pack_h2(dp[0], dp[1]), um::pack_h2(dp[2], dp[3]));
        }
        if (hsel) {                                     // direction 20: emb1 cols 4..7, emb2 cols 40, 41
          float g1[8], g2[8], c[6];
          eg_load8(0, g1);
          eg_load8(EG_E2 + 10, g2);
          um::cos_ladder(fmaf(Bd[2 * um::DIRS_PITCH + 20], t2x, fmaf(Bd[um::DIRS_PITCH + 20], t1x, Bd[20] * t0x)), c);
          float d = g1[4] * c[0];
          d = fmaf(2.f * g1[5], c[1], d); d = fmaf(4.f * g1[6], c[2], d); d = fmaf(8.f * g1[7], c[3], d);
          d = fmaf(16.f * g2[0], c[4], d); d = fmaf(32.f * g2[1], c[5], d);
          *reinterpret_cast<uint2*>(act + (FG_DPR + 2) * FGB + p * 16 + 8) = make_uint2(um::pack_h2(d * VMB_PI_F, 0.f), 0u);
        }
      }
      // dB += dproj^T [1 x y z ...]: the 21 real feature rows are in the first warpgroup's half; the second issues the
      // same instructions on rows that are never stored, which keeps the wgmma stream free of divergent branches
      OPERANDS_READY();
      mm.wgrad16(wDB, FG_DPR, FG_E1);
      MMA_DONE();
      __syncthreads();                                  // the next tile's PE overwrites E1 / E2 / DH
    }
#undef OPERANDS_READY
#undef MMA_DONE
    }   // compute threads
    if (a.fwd_only) {                                   // nothing to reduce; the weight buffer is free once every warp is done
      __syncthreads();
      if (tid == 0 && gt < gt_end) {
        ptx::mbar_arrive_expect_tx(&misc->wbar, um::IMG_BYTES);
        ptx::bulk_g2s(smem + SM_W, image + (size_t)(gt / npo) * um::IMG_BYTES, um::IMG_BYTES, &misc->wbar);
      }
      continue;
    }
    // ---- segment end: this CTA's partial sums for object b -----------------------------------------------------
    ls_d = warp_sum(ls_d); ls_c = warp_sum(ls_c); ls_o = warp_sum(ls_o);
    if (hsel == 0 && lane == 0) { float* l = misc->lsum[quad]; l[0] = ls_d; l[1] = ls_c; l[2] = ls_o; }
    __syncthreads();
    if (tid == 0 && gt < gt_end) {          // every MMA of this segment has completed: the weight buffer is free --
      ptx::mbar_arrive_expect_tx(&misc->wbar, um::IMG_BYTES);        // the next object's image lands during the flush
      ptx::bulk_g2s(smem + SM_W, image + (size_t)(gt / npo) * um::IMG_BYTES, um::IMG_BYTES, &misc->wbar);
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
    // ---- reduce + update ---------------------------------------------------------------------------------------------
    // cooperative launch: after the LAST segment (below, outside this loop), all CTAs share the reduction of all objects.
    // otherwise: the last segment of the object to arrive reduces that object's rows here.
    if (!x.cooperative) {
      __threadfence();
      __syncthreads();
      const int c_first = cta_of_pair(rg, G, b * npo), c_last = cta_of_pair(rg, G, (b + 1) * npo - 1);
      if (tid == 0) misc->fin = (atomicAdd(&x.obj_done[b], 1u) + 1u == (unsigned int)(c_last - c_first + 1)) ? 1 : 0;
      __syncthreads();
      if (misc->fin) {
        __threadfence();
        const int skip = finish_rows(b, 0, L.stride >> 2, true);
        if (tid == 0) {
          x.obj_done[b] = 0u;
          if (x.fuse_adam && x.step_counter && a.backward && !skip) x.step_counter[b] += 1;
        }
      }
    }
    __syncthreads();
  }

  if (x.cooperative && !a.fwd_only) {
    // ---- grid-wide finish: every CTA is resident (cooperative launch), all of them end their tiles within one round
    // of each other, and the reduction of ALL objects' partial rows + AdamW is split evenly over the grid (less than one
    // float4 of the parameter block per thread) instead of one object per SM on the kernel's tail.
    // gbar[0] arrive, gbar[1] depart;  x.obj_done[B + b] = skip flag of object b
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      atomicAdd(&gbar[0], 1u);
      unsigned int spins = 0;
      while (atomicAdd(&gbar[0], 0u) < (unsigned int)G) { __nanosleep(32); if (++spins > 400000000u) __trap(); }
    }
    __syncthreads();
    __threadfence();
    const int n4 = L.stride >> 2;
    const long long W = (long long)a.B * n4;
    const long long lo = (W * blockIdx.x) / G, hi = (W * (blockIdx.x + 1)) / G;
    for (int b = (int)(lo / n4); (long long)b * n4 < hi; ++b) {
      const int i_lo = (int)(max(lo, (long long)b * n4) - (long long)b * n4);
      const int i_hi = (int)(min(hi, (long long)(b + 1) * n4) - (long long)b * n4);
      const int skip = finish_rows(b, i_lo, i_hi, i_lo == 0);
      if (i_lo == 0 && tid == 0) x.obj_done[a.B + b] = (unsigned int)skip;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) misc->fin = (atomicAdd(&gbar[1], 1u) + 1u == (unsigned int)G) ? 1 : 0;
    __syncthreads();
    if (misc->fin) {                                    // the last CTA to leave: step numbers, re-arm the barrier
      __threadfence();
      if (x.fuse_adam && x.step_counter && a.backward)
        for (int b = tid; b < a.B; b += NT) if (x.obj_done[a.B + b] == 0u) x.step_counter[b] += 1;
      if (x.loss_sum && warp == 0) {                    // scalar loss of the step (loss.py:59-62), fixed summation order
        float s = 0.f;
        for (int b = lane; b < a.B; b += 32) s += __ldcg(a.loss_terms + b * 4 + 3);
        s = warp_sum(s);
        if (lane == 0) *x.loss_sum = s;
      }
      __syncthreads();
      if (tid == 0) { gbar[0] = 0u; gbar[1] = 0u; gbar[2] = 0u; gbar[3] = 0u; gbar[4] = 0u; gbar[5] = 0u; }
    }
  }

}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static int fused_rows_needed(int n_obj, int n_sm) { return n_obj + n_sm; }

// Cost-aware split of B objects x npo tile pairs over G CTAs.  Starting a second object inside a CTA costs it a flush
// of the gradient partial, a weight load and a pipeline refill, so pairs are laid out on a
// virtual axis x(p) = p + beta * (object of p) -- every object boundary is a gap of beta -- and that axis is split
// evenly: a CTA whose range crosses a boundary gets correspondingly fewer pairs.  beta is the largest of {1, 0.7, 0.4, 0}
// that does not raise the maximum number of rounds per CTA.
static void fused_partition(int B, int npo, int G, uf::Ranges& rg) {
  const long long T = (long long)B * npo;
  double beta = 0.0;
  if (T >= 2LL * G) {
    const long long rounds = (T + G - 1) / G;
    for (double cand : {1.0, 0.7, 0.4}) {
      if ((long long)std::ceil(((double)T + cand * (B - 1)) / G - 1e-9) <= rounds) { beta = cand; break; }
    }
  }
  const double V = (double)T + beta * (B - 1);
  int c = 0;
  rg.begin[0] = 0;
  for (long long p = 0; p < T; ++p) {
    const double x = (double)p + beta * (double)(p / npo);
    while (c < G - 1 && x >= V * (c + 1) / G && p > rg.begin[c] && T - p >= G - 1 - c) rg.begin[++c] = (int)p;
    if (T - p - 1 == G - 1 - c && c < G - 1) {            // one pair left per remaining CTA
      for (long long q = p + 1; q < T; ++q) rg.begin[++c] = (int)q;
      break;
    }
  }
  while (c < G) rg.begin[++c] = (int)T;
}

static int fused_launch_step(const VmbLayout& L, const StepParams& sp, const FusedExtra& fx, const void* image, int n_sm,
                             cudaStream_t st, std::string& err, bool* cooperative = nullptr) {
  using namespace uf;
  if (L.H != 32 || L.nfreq != 6) { err = "fused step kernel: hidden must be 32 and n_freq 6"; return -4; }
  if (sp.S < 1 || sp.S > 32) { err = "fused step kernel: n_samples must be in [1, 32]"; return -4; }
  if (!sp.fwd_only && sp.B > MAX_OBJ_SMEM) { err = "fused step kernel: too many objects for the in-kernel mask counts"; return -4; }
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  const int smem_bytes = SM_CNT + (sp.fwd_only ? 0 : sp.B * 12) + 16;
  if (!attr_set[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(k_step_fused<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_step_fused<10>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_step_fused<14>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
    if (e != cudaSuccess) { err = std::string("cudaFuncSetAttribute(k_step_fused): ") + cudaGetErrorString(e); return -2; }
    attr_set[dev & 63] = true;
  }
  const int rpw = 32 / sp.S;                  // whole rays per warp: the sample axis never crosses a warp
  const int nr = 4 * rpw;
  const int tpo = (sp.R + nr - 1) / nr;       // tiles per object
  const int npo = (tpo + 1) / 2;              // rounds (tile pairs) per object
  const long long T = (long long)npo * sp.B;
  if (T > 0x7fffffffLL) { err = "fused step kernel: too many tiles"; return -1; }
  long long grid = T;
  if (grid > n_sm) grid = n_sm;
  if (grid > MAX_CTAS) grid = MAX_CTAS;
  if (grid < 1) grid = 1;
  Ranges rg;
  fused_partition(sp.B, npo, (int)grid, rg);
  const unsigned char* img = (const unsigned char*)image;
  FusedExtra fxl = fx;
  // every CTA is resident (grid <= #SMs, one CTA per SM) -- the cooperative attribute makes the runtime guarantee it,
  // which is what lets an object's CTAs wait for each other in the shared reduction
  static int coop_ok[64] = {};
  if (coop_ok[dev & 63] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrCooperativeLaunch, dev);
    coop_ok[dev & 63] = v ? 1 : -1;
  }
  fxl.cooperative = (coop_ok[dev & 63] == 1 && !sp.fwd_only && getenv("VMB_NO_COOP") == nullptr) ? 1 : 0;
  if (cooperative) *cooperative = fxl.cooperative != 0;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(NT); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = fxl.cooperative;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaError_t e;
  if (sp.S == 10)      e = cudaLaunchKernelEx(&cfg, k_step_fused<10>, sp, fxl, L, img, rg, tpo, npo, nr, rpw);
  else if (sp.S == 14) e = cudaLaunchKernelEx(&cfg, k_step_fused<14>, sp, fxl, L, img, rg, tpo, npo, nr, rpw);
  else                 e = cudaLaunchKernelEx(&cfg, k_step_fused<0>, sp, fxl, L, img, rg, tpo, npo, nr, rpw);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { err = std::string("k_step_fused launch: ") + cudaGetErrorString(e); return -2; }
  return 0;
}
