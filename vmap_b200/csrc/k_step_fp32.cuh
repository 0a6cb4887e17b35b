// K1 (fp32 flavour): fused PE -> MLP -> volume render -> loss -> backward for a stack of
// per-object MLPs, CUDA-core fp32 throughout.  Any hidden size; this is the parity anchor
// (<= ~1e-5 rel-L2 vs the reference's fp32 functorch path) and the path used for the
// H=128 background model and the H=256 iMAP model.  The H=32 fast path is k_step_fused.cuh.
//
// Reference arithmetic restated here:
//   embedding.py:82-91  (UniDirsEmbed.forward)      model.py:54-85   (OccupancyMap.forward)
//   render_rays.py:4-8,26-34,47-51 (sigmoid, termination, render)
//   loss.py:5-62 + render_rays.py:53-96 (masked L1 losses, 1/(sqrt(var)+1e-4) weighting)
//   and the autograd backward of all of it (train.py:324).
//
// One CTA = one tile of whole rays of one object; the network on the tile (NetTile below) is
// shared with K10 / K11 (k_track.cuh).  dY_l overwrites h_l in place once wgrad_{l+1} has
// consumed h_l.
#pragma once
#include "common.cuh"

struct StepParams {
  int B, R, S;
  const float* pcs;  long long pcs_stride;
  const float* z;    long long z_stride;
  const float* gt_depth;  long long gt_depth_stride;
  const float* gt_colour; long long gt_colour_stride;
  const unsigned char* sem;  long long sem_stride;
  const unsigned char* mask; long long mask_stride;
  const float* params;
  const float* scale;
  float* grads;
  float* loss_terms;
  float* r_depth; float* r_var; float* r_colour; float* r_opacity;
  const int* counts;            // [B][4]
  float cs, os;
  int backward;
  // forward-only mode (vmb_forward): S == 1, R == n_points
  int fwd_only;
  float* out_alpha;  long long alpha_stride;
  float* out_colour; long long colour_stride;
};

// the mask counts of a slice of rays (loss.py:16-18,38), one ray's increment: depth (mask and object), object, not-unknown
__device__ __forceinline__ void slice_mask_count(const unsigned char* sem, const unsigned char* mask, int r, int& nd,
                                                 int& no, int& ns) {
  const int s = sem[r];
  const int mo = s != 0;
  nd += (mask[r] != 0) & mo; no += mo; ns += s != 2;
}

// the warp sums of the three counts (K0, K10 / K11): lane 0 of warp w writes red[0..2][w]; tid = threadIdx.x, as the
// caller holds it (unsigned or int)
template <class Tid, int NW>
__device__ __forceinline__ void warp_mask_counts(Tid tid, int nd, int no, int ns, int (&red)[3][NW]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nd += __shfl_xor_sync(0xffffffffu, nd, o);
    no += __shfl_xor_sync(0xffffffffu, no, o);
    ns += __shfl_xor_sync(0xffffffffu, ns, o);
  }
  if ((tid & 31) == 0) { red[0][tid >> 5] = nd; red[1][tid >> 5] = no; red[2][tid >> 5] = ns; }
}

// ---------------------------------------------------------------------------------------
// K0: per-object mask counts N_d = sum(mask_depth & sem!=0), N_o = sum(sem!=0),
// N_s = sum(sem!=2)  (loss.py:16-18,38; render_rays.py:68,86).  Also clears loss_terms.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_mask_counts(int R, const unsigned char* sem, long long sem_stride,
                                                      const unsigned char* mask, long long mask_stride,
                                                      int* counts, float* loss_terms) {
  const int b = blockIdx.x;
  const unsigned char* s = sem + (size_t)b * sem_stride;
  const unsigned char* m = mask + (size_t)b * mask_stride;
  int nd = 0, no = 0, ns = 0;
  for (int r = threadIdx.x; r < R; r += blockDim.x) slice_mask_count(s, m, r, nd, no, ns);
  __shared__ int red[3][8];
  warp_mask_counts(threadIdx.x, nd, no, ns, red);
  __syncthreads();
  if (threadIdx.x < 3) {
    int t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[threadIdx.x][w];
    counts[b * 4 + threadIdx.x] = t;
  }
  if (threadIdx.x == 3) counts[b * 4 + 3] = 0;
  if (loss_terms != nullptr && threadIdx.x < 4) loss_terms[b * 4 + threadIdx.x] = 0.f;
}

// ---------------------------------------------------------------------------------------
// dense helpers
// ---------------------------------------------------------------------------------------
// acc[j] += sum_k W[j*ld + k] * x[k*PT]     (W -> row o, column c0 of a [out][in] matrix)
// W steps one column per k: the row addresses stay loop-invariant offsets of one pointer
// (fewer address instructions per FMA than indexing W + j*ld + k in the inlined loops).
template <int OB>
__device__ __forceinline__ void fwd_block(float (&acc)[OB], const float* __restrict__ W, int ld,
                                          const float* x, int K, int PT) {
  for (int k = 0; k < K; ++k, ++W) {
    const float xv = x[k * PT];
#pragma unroll
    for (int j = 0; j < OB; ++j) acc[j] = fmaf(__ldg(W + j * ld), xv, acc[j]);
  }
}
// acc[j] += sum_o dy[o*PT] * W[o*ld + j]    (W -> row 0, column k of a [out][in] matrix)
template <int OB>
__device__ __forceinline__ void dgrad_block(float (&acc)[OB], const float* __restrict__ W, int ld,
                                            const float* dy, int H, int PT) {
  for (int o = 0; o < H; ++o) {
    const float d = dy[o * PT];
#pragma unroll
    for (int j = 0; j < OB; ++j) acc[j] = fmaf(d, __ldg(W + o * ld + j), acc[j]);
  }
}

// ---------------------------------------------------------------------------------------
// The network on one tile, written once for K1 fp32 and K10 / K11 (k_track.cuh), so the
// pose gradient is the gradient of the network the step trains.
// One CTA (NT threads) = one tile of `nr` whole rays (np = nr*S <= TP points) of one object;
// thread tid works on point p = tid % TP and on the OPT output features from o_lo of its
// group og = tid / TP.  Activations live in shared memory as [feature][point] with a +1
// pitch, so the thread-per-point phases (forward, dgrad) and the thread-per-weight phase
// (wgrad) are both bank-conflict free.  Each phase below ends with __syncthreads().
// ---------------------------------------------------------------------------------------
template <int H, int TP>
struct NetTile {
  static constexpr int NT = 128;
  static constexpr int PT = TP + 1;
  static constexpr int NOG = NT / TP;     // threads cooperating on one point
  static constexpr int OPT = H / NOG;     // output features per thread
  static constexpr int OB = 8;
  static_assert(OPT % OB == 0, "feature split must be a multiple of the register block");

  float* sE;                              // [E][PT]   rows 0..2 = network input t, then sin features
  float* sA1;                             // fc1 / dY1
  float* sA2;                             // fc2 / dY2
  float* sA3;                             // fc3 / dY3
  float* sA4;                             // fc4 / dY4
  float* sAC;                             // colour hidden / dYc
  float* sHd;                             // 12 rows: alpha, col0..2, d_araw, d_rc0..2, z, occ, T, w
  int p, og;
  int nr, np, r0;                         // whole rays per tile, points per tile, first ray
  int rl, sidx;                           // ray of the tile and sample of point p
  bool pvalid;
  int o_lo;

  __device__ __forceinline__ NetTile(float* sm, const VmbLayout& L, int S, int R)
      : sE(sm), sA1(sE + L.E * PT), sA2(sA1 + H * PT), sA3(sA2 + H * PT), sA4(sA3 + H * PT), sAC(sA4 + H * PT),
        sHd(sAC + H * PT), p((int)threadIdx.x % TP), og((int)threadIdx.x / TP), nr(TP / S), np(nr * S),
        r0(blockIdx.x * nr), rl(p / S), sidx(p - rl * S), pvalid((p < np) && (r0 + rl < R)), o_lo(og * OPT) {}

  // host: dynamic shared memory of the carve above plus `extra_rows` rows of the kernel's own after sHd
  static size_t smem(const VmbLayout& L, int extra_rows) {
    return sizeof(float) * (size_t)(L.E + 5 * H + 12 + extra_rows) * PT;
  }

  // positional embedding (embedding.py:82-91): the sin rows of sE from the network input t
  // (rows 0..2, which the kernel writes)
  __device__ __forceinline__ void embed(const float* __restrict__ P, const VmbLayout& L, float3 t) const {
    for (int d = og; d < VMB_NDIRS; d += NOG) {
      const float* Bd = P + L.o_B + d * 3;
      const float proj = fmaf(__ldg(Bd + 2), t.z, fmaf(__ldg(Bd + 1), t.y, __ldg(Bd) * t.x));
      for (int k = 0; k < L.nfreq; ++k) sE[(3 + k * VMB_NDIRS + d) * PT + p] = sinf((proj * (float)(1 << k)) * VMB_PI_F);
    }
    __syncthreads();
  }

  // MLP forward (model.py:54-85): fc1..fc4, colour hidden, raw alpha * 10 and sigmoid colour into sHd rows 0..3
  __device__ __forceinline__ void forward(const float* __restrict__ P, const VmbLayout& L) const {
    // in_layer: emb1 -> fc1
    for (int o = o_lo; o < o_lo + OPT; o += OB) {
      float acc[OB];
#pragma unroll
      for (int j = 0; j < OB; ++j) acc[j] = __ldg(P + L.o_bin + o + j);
      fwd_block<OB>(acc, P + L.o_Win + o * VMB_E1, VMB_E1, sE + p, VMB_E1, PT);
#pragma unroll
      for (int j = 0; j < OB; ++j) sA1[(o + j) * PT + p] = fmaxf(acc[j], 0.f);
    }
    __syncthreads();
    // mid1: fc1 -> fc2
    for (int o = o_lo; o < o_lo + OPT; o += OB) {
      float acc[OB];
#pragma unroll
      for (int j = 0; j < OB; ++j) acc[j] = __ldg(P + L.o_bm1 + o + j);
      fwd_block<OB>(acc, P + L.o_Wm1 + o * H, H, sA1 + p, H, PT);
#pragma unroll
      for (int j = 0; j < OB; ++j) sA2[(o + j) * PT + p] = fmaxf(acc[j], 0.f);
    }
    __syncthreads();
    // cat_layer: [fc2, emb1] -> fc3
    {
      const int ld = H + VMB_E1;
      for (int o = o_lo; o < o_lo + OPT; o += OB) {
        float acc[OB];
#pragma unroll
        for (int j = 0; j < OB; ++j) acc[j] = __ldg(P + L.o_bcat + o + j);
        fwd_block<OB>(acc, P + L.o_Wcat + o * ld, ld, sA2 + p, H, PT);
        fwd_block<OB>(acc, P + L.o_Wcat + o * ld + H, ld, sE + p, VMB_E1, PT);
#pragma unroll
        for (int j = 0; j < OB; ++j) sA3[(o + j) * PT + p] = fmaxf(acc[j], 0.f);
      }
    }
    __syncthreads();
    // mid2: fc3 -> fc4
    for (int o = o_lo; o < o_lo + OPT; o += OB) {
      float acc[OB];
#pragma unroll
      for (int j = 0; j < OB; ++j) acc[j] = __ldg(P + L.o_bm2 + o + j);
      fwd_block<OB>(acc, P + L.o_Wm2 + o * H, H, sA3 + p, H, PT);
#pragma unroll
      for (int j = 0; j < OB; ++j) sA4[(o + j) * PT + p] = fmaxf(acc[j], 0.f);
    }
    __syncthreads();
    // color_linear: [fc4, emb2] -> hc ; out_alpha: fc4 -> alpha*10
    {
      const int ld = H + L.e2;
      for (int o = o_lo; o < o_lo + OPT; o += OB) {
        float acc[OB];
#pragma unroll
        for (int j = 0; j < OB; ++j) acc[j] = __ldg(P + L.o_bcl + o + j);
        fwd_block<OB>(acc, P + L.o_Wcl + o * ld, ld, sA4 + p, H, PT);
        fwd_block<OB>(acc, P + L.o_Wcl + o * ld + H, ld, sE + VMB_E1 * PT + p, L.e2, PT);
#pragma unroll
        for (int j = 0; j < OB; ++j) sAC[(o + j) * PT + p] = fmaxf(acc[j], 0.f);
      }
      if (og == 0) {
        float acc1[1] = {__ldg(P + L.o_ba)};
        fwd_block<1>(acc1, P + L.o_Wa, H, sA4 + p, H, PT);
        sHd[0 * PT + p] = acc1[0] * 10.0f;                  // model.py:77
      }
    }
    __syncthreads();
    if (og == 0) {                                          // out_color + sigmoid (model.py:82-83)
      float acc3[3] = {__ldg(P + L.o_boc), __ldg(P + L.o_boc + 1), __ldg(P + L.o_boc + 2)};
      fwd_block<3>(acc3, P + L.o_Woc, H, sAC + p, H, PT);
#pragma unroll
      for (int c = 0; c < 3; ++c) sHd[(1 + c) * PT + p] = vmb_sigmoid(acc3[c]);
    }
    __syncthreads();
  }

  // input gradients, each in place of the activation it differentiates, from d_araw and d_rawc (sHd rows 4..7)

  // dYc = relu'(hc) * (d_rawc @ W_oc)
  __device__ __forceinline__ void dyc(const float* __restrict__ P, const VmbLayout& L) const {
    for (int o = o_lo; o < o_lo + OPT; ++o) {
      float v = sHd[5 * PT + p] * __ldg(P + L.o_Woc + o);
      v = fmaf(sHd[6 * PT + p], __ldg(P + L.o_Woc + H + o), v);
      v = fmaf(sHd[7 * PT + p], __ldg(P + L.o_Woc + 2 * H + o), v);
      sAC[o * PT + p] = (sAC[o * PT + p] > 0.f) ? v : 0.f;
    }
    __syncthreads();
  }

  // dY4 = relu'(fc4) * (dYc @ W_cl[:, :H] + d_araw * W_a)
  __device__ __forceinline__ void dy4(const float* __restrict__ P, const VmbLayout& L) const {
    const int ld = H + L.e2;
    for (int k = o_lo; k < o_lo + OPT; k += OB) {
      float acc[OB];
      const float da = sHd[4 * PT + p];
#pragma unroll
      for (int j = 0; j < OB; ++j) acc[j] = da * __ldg(P + L.o_Wa + k + j);
      dgrad_block<OB>(acc, P + L.o_Wcl + k, ld, sAC + p, H, PT);
#pragma unroll
      for (int j = 0; j < OB; ++j) sA4[(k + j) * PT + p] = (sA4[(k + j) * PT + p] > 0.f) ? acc[j] : 0.f;
    }
    __syncthreads();
  }

  // dX = relu'(X) * (dY @ W[:, :H]) for the layer X -> Y with weights W ([H][ld]): dY3, dY2, dY1
  __device__ __forceinline__ void dgrad(float* sX, const float* sDY, const float* __restrict__ W, int ld) const {
    for (int k = o_lo; k < o_lo + OPT; k += OB) {
      float acc[OB];
#pragma unroll
      for (int j = 0; j < OB; ++j) acc[j] = 0.f;
      dgrad_block<OB>(acc, W + k, ld, sDY + p, H, PT);
#pragma unroll
      for (int j = 0; j < OB; ++j) sX[(k + j) * PT + p] = (sX[(k + j) * PT + p] > 0.f) ? acc[j] : 0.f;
    }
    __syncthreads();
  }
};

// gW[o*ld + k] += sum_p dY[o][p] * X[k][p]   for o < H, k < K   (atomic: several tiles per object)
template <int H>
__device__ __forceinline__ void wgrad_part(const float* dY, const float* X, int K, float* gW, int ld,
                                           int np, int PT) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int ob = warp * 4; ob < H; ob += 16) {
    for (int kc = 0; kc < K; kc += 128) {
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      int kk[4]; bool ok[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { kk[j] = kc + lane + 32 * j; ok[j] = kk[j] < K; if (!ok[j]) kk[j] = 0; }
      for (int p = 0; p < np; ++p) {
        float dy[4], x[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) dy[i] = dY[(ob + i) * PT + p];
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = X[kk[j] * PT + p];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(dy[i], x[j], acc[i][j]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (ok[j]) atomicAdd(gW + (size_t)(ob + i) * ld + kk[j], acc[i][j]);
    }
  }
}

template <int H>
__device__ __forceinline__ void bias_grad(const float* dY, float* gb, int np, int PT) {
  for (int o = threadIdx.x; o < H; o += blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < np; ++p) s += dY[o * PT + p];
    atomicAdd(gb + o, s);
  }
}

// ---------------------------------------------------------------------------------------
// K1 fp32
// ---------------------------------------------------------------------------------------
template <int H, int TP>
__global__ void __launch_bounds__(128) k_step_fp32(StepParams a, VmbLayout L) {
  using Net = NetTile<H, TP>;
  constexpr int NT = Net::NT, PT = Net::PT, NOG = Net::NOG;
  extern __shared__ float sm[];
  const Net net(sm, L, a.S, a.R);
  float* sDp = net.sHd + 12 * PT;         // [21][PT] d(loss)/d(proj)
  __shared__ int s_on[3];
  __shared__ float s_loss[4];

  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int S = a.S, R = a.R;
  const float* __restrict__ P = a.params + (size_t)b * L.stride;
  float* G = a.grads ? a.grads + (size_t)b * L.stride : nullptr;

  if (tid < 3) {
    int on = 1;
    if (!a.fwd_only) for (int i = 0; i < a.B; ++i) on &= (a.counts[i * 4 + tid] != 0);
    s_on[tid] = on;                       // render_rays.py:68-73: any empty mask zeroes the term for all
  }
  if (tid < 4) s_loss[tid] = 0.f;

  // ---- A: load point, positional embedding (embedding.py:82-91) -----------------------
  float3 t = make_float3(0.f, 0.f, 0.f);
  if (net.pvalid) {
    const size_t gi = (size_t)b * a.pcs_stride + ((size_t)(net.r0 + net.rl) * S + net.sidx) * 3;
    const float sc = a.scale[b];
    t.x = a.pcs[gi] / sc; t.y = a.pcs[gi + 1] / sc; t.z = a.pcs[gi + 2] / sc;
  }
  if (net.og == 0) {
    const int p = net.p;
    net.sE[0 * PT + p] = t.x; net.sE[1 * PT + p] = t.y; net.sE[2 * PT + p] = t.z;
    net.sHd[8 * PT + p] = (net.pvalid && !a.fwd_only) ? a.z[(size_t)b * a.z_stride + (size_t)(net.r0 + net.rl) * S + net.sidx] : 0.f;
    net.sHd[4 * PT + p] = 0.f; net.sHd[5 * PT + p] = 0.f; net.sHd[6 * PT + p] = 0.f; net.sHd[7 * PT + p] = 0.f;
  }
  net.embed(P, L, t);

  // ---- B: MLP forward (model.py:54-85) -------------------------------------------------
  net.forward(P, L);

  if (a.fwd_only) {
    if (net.og == 0 && net.pvalid) {
      const size_t n = (size_t)(net.r0 + net.rl);
      a.out_alpha[(size_t)b * a.alpha_stride + n] = net.sHd[0 * PT + net.p];
      float* oc = a.out_colour + (size_t)b * a.colour_stride + n * 3;
      oc[0] = net.sHd[1 * PT + net.p]; oc[1] = net.sHd[2 * PT + net.p]; oc[2] = net.sHd[3 * PT + net.p];
    }
    return;
  }

  // ---- C: volume render + loss + d(loss)/d(alpha, colour)  (render_rays.py, loss.py) ---
  float l_d = 0.f, l_c = 0.f, l_o = 0.f;
  if (tid < net.nr && net.r0 + tid < R) {
    const int ray = net.r0 + tid;
    const int pb = tid * S;
    float T = 1.f, D = 0.f, O = 0.f, C0 = 0.f, C1 = 0.f, C2 = 0.f;
    for (int s = 0; s < S; ++s) {
      const int q = pb + s;
      const float occ = vmb_sigmoid(net.sHd[0 * PT + q]);       // render_rays.py:6
      const float w = occ * T;                              // render_rays.py:34
      net.sHd[9 * PT + q] = occ; net.sHd[10 * PT + q] = T; net.sHd[11 * PT + q] = w;
      const float zz = net.sHd[8 * PT + q];
      D = fmaf(w, zz, D); O += w;
      C0 = fmaf(w, net.sHd[1 * PT + q], C0); C1 = fmaf(w, net.sHd[2 * PT + q], C1); C2 = fmaf(w, net.sHd[3 * PT + q], C2);
      T *= (1.f - occ + 1e-10f);                            // render_rays.py:29
    }
    float V = 0.f;
    for (int s = 0; s < S; ++s) {
      const float dz = net.sHd[8 * PT + pb + s] - D;
      V = fmaf(net.sHd[11 * PT + pb + s], dz * dz, V);          // loss.py:28-29 (detached)
    }
    if (a.r_depth) a.r_depth[(size_t)b * R + ray] = D;
    if (a.r_var) a.r_var[(size_t)b * R + ray] = V;
    if (a.r_opacity) a.r_opacity[(size_t)b * R + ray] = O;
    if (a.r_colour) { float* rc = a.r_colour + ((size_t)b * R + ray) * 3; rc[0] = C0; rc[1] = C1; rc[2] = C2; }

    const int sv = a.sem[(size_t)b * a.sem_stride + ray];
    const float m_o = (sv != 0) ? 1.f : 0.f;                // loss.py:16
    const float m_s = (sv != 2) ? 1.f : 0.f;                // loss.py:18
    const float m_d = (a.mask[(size_t)b * a.mask_stride + ray] != 0) ? m_o : 0.f;   // loss.py:38
    const float gd = a.gt_depth[(size_t)b * a.gt_depth_stride + ray];
    const float* gc = a.gt_colour + (size_t)b * a.gt_colour_stride + (size_t)ray * 3;
    const float inv_nd = 1.f / ((float)a.counts[b * 4 + 0] + 1e-10f);
    const float inv_no = 1.f / ((float)a.counts[b * 4 + 1] + 1e-10f);
    const float inv_ns = 1.f / ((float)a.counts[b * 4 + 2] + 1e-10f);
    const float info = 1.f / (sqrtf(V) + 1e-4f);            // render_rays.py:74-79
    const float on_d = s_on[0] ? 1.f : 0.f, on_c = s_on[1] ? 1.f : 0.f, on_o = s_on[2] ? 1.f : 0.f;
    const float e_d = D - gd, e_o = O - m_o;
    const float e_c0 = C0 - gc[0], e_c1 = C1 - gc[1], e_c2 = C2 - gc[2];
    l_d = on_d * fabsf(e_d) * m_d * info * inv_nd;
    l_c = on_c * (fabsf(e_c0) + fabsf(e_c1) + fabsf(e_c2)) * m_o * inv_no;
    l_o = on_o * fabsf(e_o) * m_s * inv_ns;
    if (a.backward) {
      const float gD = on_d * vmb_sign(e_d) * m_d * info * inv_nd;
      const float kc = on_c * a.cs * m_o * inv_no;
      const float gC0 = kc * vmb_sign(e_c0), gC1 = kc * vmb_sign(e_c1), gC2 = kc * vmb_sign(e_c2);
      const float gO = on_o * a.os * vmb_sign(e_o) * m_s * inv_ns;
      float suffix = 0.f;                                    // sum_{k>s} G_k w_k
      for (int s = S - 1; s >= 0; --s) {
        const int q = pb + s;
        const float occ = net.sHd[9 * PT + q], Ts = net.sHd[10 * PT + q], w = net.sHd[11 * PT + q];
        const float c0 = net.sHd[1 * PT + q], c1 = net.sHd[2 * PT + q], c2 = net.sHd[3 * PT + q];
        const float Gs = fmaf(gD, net.sHd[8 * PT + q], fmaf(gC0, c0, fmaf(gC1, c1, fmaf(gC2, c2, gO))));
        const float f = 1.f - occ + 1e-10f;
        const float docc = Gs * Ts - suffix / f;
        net.sHd[4 * PT + q] = 10.0f * docc * occ * (1.f - occ);  // d/d(raw alpha), model.py:77
        net.sHd[5 * PT + q] = gC0 * w * c0 * (1.f - c0);         // d/d(raw colour) through sigmoid
        net.sHd[6 * PT + q] = gC1 * w * c1 * (1.f - c1);
        net.sHd[7 * PT + q] = gC2 * w * c2 * (1.f - c2);
        suffix = fmaf(Gs, w, suffix);
      }
    }
  }
  // per-object loss terms
  l_d = warp_sum(l_d); l_c = warp_sum(l_c); l_o = warp_sum(l_o);
  if ((tid & 31) == 0) {
    atomicAdd(&s_loss[0], l_d); atomicAdd(&s_loss[1], l_c); atomicAdd(&s_loss[2], l_o);
  }
  __syncthreads();
  if (tid < 3 && a.loss_terms) atomicAdd(a.loss_terms + b * 4 + tid, s_loss[tid]);
  if (tid == 3 && a.loss_terms) atomicAdd(a.loss_terms + b * 4 + 3, s_loss[0] + a.cs * s_loss[1] + a.os * s_loss[2]);
  if (!a.backward) return;

  // ---- D: backward ---------------------------------------------------------------------
  // heads: dW_a, db_a, dW_oc, db_oc
  for (int idx = tid; idx < 4 * H; idx += NT) {
    const int c = idx / H, o = idx - c * H;
    const float* x = (c == 0) ? net.sA4 : net.sAC;
    const float* dy = net.sHd + (4 + c) * PT;
    float s = 0.f;
    for (int q = 0; q < net.np; ++q) s = fmaf(dy[q], x[o * PT + q], s);
    atomicAdd(G + (c == 0 ? L.o_Wa + o : L.o_Woc + (c - 1) * H + o), s);
  }
  if (tid < 4) {
    float s = 0.f;
    for (int q = 0; q < net.np; ++q) s += net.sHd[(4 + tid) * PT + q];
    atomicAdd(G + (tid == 0 ? L.o_ba : L.o_boc + tid - 1), s);
  }
  __syncthreads();
  net.dyc(P, L);
  {   // color_linear wgrad: X = [fc4 | emb2]
    const int ld = H + L.e2;
    wgrad_part<H>(net.sAC, net.sA4, H, G + L.o_Wcl, ld, net.np, PT);
    wgrad_part<H>(net.sAC, net.sE + VMB_E1 * PT, L.e2, G + L.o_Wcl + H, ld, net.np, PT);
    bias_grad<H>(net.sAC, G + L.o_bcl, net.np, PT);
  }
  __syncthreads();
  net.dy4(P, L);
  wgrad_part<H>(net.sA4, net.sA3, H, G + L.o_Wm2, H, net.np, PT);          // mid2 wgrad
  bias_grad<H>(net.sA4, G + L.o_bm2, net.np, PT);
  __syncthreads();
  net.dgrad(net.sA3, net.sA4, P + L.o_Wm2, H);                              // dY3
  {   // cat_layer wgrad: X = [fc2 | emb1]
    const int ld = H + VMB_E1;
    wgrad_part<H>(net.sA3, net.sA2, H, G + L.o_Wcat, ld, net.np, PT);
    wgrad_part<H>(net.sA3, net.sE, VMB_E1, G + L.o_Wcat + H, ld, net.np, PT);
    bias_grad<H>(net.sA3, G + L.o_bcat, net.np, PT);
  }
  __syncthreads();
  net.dgrad(net.sA2, net.sA3, P + L.o_Wcat, H + VMB_E1);                    // dY2
  wgrad_part<H>(net.sA2, net.sA1, H, G + L.o_Wm1, H, net.np, PT);          // mid1 wgrad
  bias_grad<H>(net.sA2, G + L.o_bm1, net.np, PT);
  __syncthreads();
  net.dgrad(net.sA1, net.sA2, P + L.o_Wm1, H);                              // dY1
  wgrad_part<H>(net.sA1, net.sE, VMB_E1, G + L.o_Win, VMB_E1, net.np, PT); // in_layer wgrad
  bias_grad<H>(net.sA1, G + L.o_bin, net.np, PT);

  // PE backward: d/d(proj_d) = sum_k g_emb[3+k*21+d] * cos(arg) * pi * 2^k ; dB = dproj^T t
  {
    const int ldc = H + VMB_E1, ldl = H + L.e2;
    for (int d = net.og; d < VMB_NDIRS; d += NOG) {
      const float* Bd = P + L.o_B + d * 3;
      const float proj = fmaf(__ldg(Bd + 2), t.z, fmaf(__ldg(Bd + 1), t.y, __ldg(Bd) * t.x));
      float dp = 0.f;
      for (int k = 0; k < L.nfreq; ++k) {
        const int j = 3 + k * VMB_NDIRS + d;
        float g = 0.f;
        if (j < VMB_E1) {
          for (int o = 0; o < H; ++o) {
            g = fmaf(net.sA1[o * PT + net.p], __ldg(P + L.o_Win + o * VMB_E1 + j), g);
            g = fmaf(net.sA3[o * PT + net.p], __ldg(P + L.o_Wcat + o * ldc + H + j), g);
          }
        } else {
          for (int o = 0; o < H; ++o) g = fmaf(net.sAC[o * PT + net.p], __ldg(P + L.o_Wcl + o * ldl + H + (j - VMB_E1)), g);
        }
        const float fk = (float)(1 << k);
        const float arg = (proj * fk) * VMB_PI_F;
        dp = fmaf(g * cosf(arg) * VMB_PI_F, fk, dp);
      }
      sDp[d * PT + net.p] = dp;
    }
  }
  __syncthreads();
  if (tid < VMB_NDIRS * 3) {
    const int d = tid / 3, i = tid - d * 3;
    float s = 0.f;
    for (int q = 0; q < net.np; ++q) s = fmaf(sDp[d * PT + q], net.sE[i * PT + q], s);
    atomicAdd(G + L.o_B + tid, s);
  }
}
