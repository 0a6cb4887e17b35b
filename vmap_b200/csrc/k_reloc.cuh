// Relocalisation against the object map: the tracking loss of many candidate poses of one frame in one launch, and the
// top K of them, on the device.  Hidden 32 only, on the fused wgmma tile of k_track_fused.cuh.
//
// The rule is K10's loss (k_track.cuh) at each hypothesis T_h of the table hyps [n_hyp][4][4] (fp64 T_wc):
//   Samples  the frame's camera-frame points q of one ray slice (the tracker's own draw), shared by every hypothesis:
//            nothing is sampled per hypothesis.  The mask counts depend on the pixels only, so each CTA counts its
//            object's once and every hypothesis it scores uses them.
//   Forward  load_object, forward_tile and render_ray of k_track_fused.cuh: pose_point with T_h, E0 and the six forward
//            wgmma stages from the object's fp16 image row, the heads, the fp64 render and ray_loss (per-object,
//            per-term empty masks, weights 1 / colour_scaling / opacity_scaling).  No input-gradient chain, no pose
//            terms.  One CTA = one fused tile of one object (blockIdx.y) and a chunk of hypotheses (blockIdx.z): the
//            weight image, the mask counts and the sample tile stay in shared memory / registers across the chunk.
//   Reduce   per (hypothesis, object) in K10's order: each ray's three loss terms, rays in order within each
//            vmb_track_tiles tile (128 / S rays), tiles in order, total = L_d + cs L_c + os L_o, then over the group's
//            objects by vmb_track_update's fixed tree.  So on one group the score at T is, bit for bit, the loss the
//            tracker reports for an iteration run from T on the same slice.  scores[h] += that sum: several groups
//            accumulate in call order (the tracker joins all groups' objects in one tree, so with more than one group
//            the two differ in the last bits).  No floating-point atomics: bitwise reproducible, and a hypothesis's
//            score does not depend on n_hyp or the chunking.
//   Select   k_reloc_select: the rank of every score, ascending, ties to the lower index, non-finite scores after
//            every finite one (in index order); the K first indices and their poses.
// Registers (ptxas -v, sm_90a), no spills: k_reloc_fused 98; k_reloc_reduce 40; k_reloc_select 32.
// Shared memory per CTA of k_reloc_fused: k_track_fused's layout (tf::SMEM), so two CTAs share an SM.
#pragma once
#include "k_track_fused.cuh"

namespace rl {

constexpr int NT = tf::NT;

// per-(hypothesis, object, ray) loss terms [n_hyp][B][R][3] before K10's tile sums, sized by the call's n_hyp B R:
// handle scratch (DeviceBuffer's rule), so after a capture a larger call is refused (VMB_E_CUDA): run the largest shape
// eagerly before capturing
struct Workspace {
  DeviceBuffer<double> lray;
};

// One CTA = fused tile blockIdx.x of object blockIdx.y, hypotheses [blockIdx.z * chunk, +chunk) of n_hyp.
// nr = 4 rpw rays per tile, rpw = 32 / S rays per warp.  lray: [n_hyp][B][R][3].
__global__ void __launch_bounds__(NT, 2) k_reloc_fused(TrackParams a, const unsigned char* __restrict__ image,
                                                       const double* __restrict__ hyps, int n_hyp, int chunk, int nr,
                                                       int rpw, double* __restrict__ lray) {
  using namespace tf;
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ int red[3][NT / 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.y, S = a.S, R = a.R, B = a.B;
  const int h0 = blockIdx.z * chunk, h1 = min(n_hyp, h0 + chunk);
  const int p = tid & 127, hsel = tid >> 7, quad = warp & 3;
  const int rw = lane / S, sidx = lane - rw * S, seg_lo = lane - sidx;
  const int ray = blockIdx.x * nr + quad * rpw + rw;
  const bool live = rw < rpw && ray < R;
  const int row = a.rows[b];
  if (row < 0 || row >= a.n_rows) {                   // uniform over the CTA: the object contributes nothing
    if (hsel == 0 && live && sidx == 0)
      for (int h = h0; h < h1; ++h)
        for (int c = 0; c < 3; ++c) lray[(((size_t)h * B + b) * R + ray) * 3 + c] = 0.0;
    if (tid == 0 && a.status) atomicOr(a.status, VMB_TRACK_ST_BAD_ROW);
    return;
  }
  const uf::Tile tl = load_object(smem, image, row, a, red, quad);
  const float sc = a.scale[row];
  float3 q = make_float3(0.f, 0.f, 0.f);
  if (live) {
    const size_t gi = (size_t)b * a.pcs_stride + ((size_t)ray * S + sidx) * 3;
    q = make_float3(a.pcs[gi], a.pcs[gi + 1], a.pcs[gi + 2]);
  }
  float zv = 0.f;
  if (hsel == 0 && live) zv = a.z[(size_t)b * a.z_stride + (size_t)ray * S + sidx];

  image_ready(smem);

  // No barrier closes an iteration: after the heads barrier only warpgroup 0's render reads shared memory, and only
  // the heads tile, which the next iteration writes after forward_tile's own barrier.
#pragma unroll 1
  for (int h = h0; h < h1; ++h) {
    const uf::PeIn tin(live ? pose_point(hyps + (size_t)h * 16, q, sc) : make_float3(0.f, 0.f, 0.f));
    uint32_t ua[8];
    forward_tile(tl, tin, ua);
    __syncthreads();                                  // heads tile (fragment layout -> point layout); mask counts
    if (hsel == 0) {                                  // warp-uniform
      const RayRender rr = render_ray(tl.hd, tl.wf, zv, p, S, sidx, seg_lo);
      int cnt[3];
      red_counts(red, cnt);
      if (live && sidx == 0) {
        const RayLoss ls = ray_loss(rr.D, rr.O, rr.C0, rr.C1, rr.C2, rr.V, a.sem[(size_t)b * a.sem_stride + ray],
                                    a.mask[(size_t)b * a.mask_stride + ray] != 0,
                                    a.gt_depth[(size_t)b * a.gt_depth_stride + ray],
                                    a.gt_colour + (size_t)b * a.gt_colour_stride + (size_t)ray * 3, true, cnt, a.cs, a.os);
        double* o = lray + (((size_t)h * B + b) * R + ray) * 3;
        o[0] = ls.l[0]; o[1] = ls.l[1]; o[2] = ls.l[2];
      }
    }
  }
}

// One CTA per hypothesis: vmb_track_update's loss sum.  Thread k takes objects k, k + 256, ... in order, each object's
// K10 tiles (nr10 rays) in order, each tile's rays in order (k_tf_reduce's rule); a fixed tree joins the threads.
__global__ void __launch_bounds__(256) k_reloc_reduce(int B, int R, int nr10, double cs, double os,
                                                      const double* __restrict__ lray, double* __restrict__ scores,
                                                      double* __restrict__ terms) {
  __shared__ double s_acc[256];
  const int tid = threadIdx.x;
  const size_t h = blockIdx.x;
  double acc = 0.0;
  for (int ob = tid; ob < B; ob += 256) {
    const double* lr = lray + (h * B + ob) * (size_t)R * 3;
    double s[3] = {0.0, 0.0, 0.0};
    for (int r0 = 0; r0 < R; r0 += nr10) {
      double t[3] = {0.0, 0.0, 0.0};
      const int r1 = min(R, r0 + nr10);
      for (int r = r0; r < r1; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) t[c] += lr[(size_t)r * 3 + c];
#pragma unroll
      for (int c = 0; c < 3; ++c) s[c] += t[c];
    }
    const double tot = s[0] + cs * s[1] + os * s[2];
    if (terms) {
      double* o = terms + (h * B + ob) * 4;
      o[0] = s[0]; o[1] = s[1]; o[2] = s[2]; o[3] = tot;
    }
    acc += tot;
  }
  s_acc[tid] = acc;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (tid < st) s_acc[tid] += s_acc[tid + st];
    __syncthreads();
  }
  if (tid == 0) scores[h] += s_acc[0];
}

// the rank of score i among n: finite scores ascending, ties to the lower index, then the non-finite ones by index
__global__ void __launch_bounds__(256) k_reloc_select(int n, const double* __restrict__ scores,
                                                      const double* __restrict__ hyps, int k, int* __restrict__ idx,
                                                      double* __restrict__ poses) {
  extern __shared__ double s_sc[];
  for (int j = threadIdx.x; j < n; j += blockDim.x) s_sc[j] = scores[j];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double si = s_sc[i];
  const bool fi = isfinite(si);
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const double sj = s_sc[j];
    const bool fj = isfinite(sj);
    rank += fi ? (fj && (sj < si || (sj == si && j < i))) : (fj || j < i);
  }
  if (rank >= k) return;
  idx[rank] = i;
  if (poses)
    for (int c = 0; c < 16; ++c) poses[(size_t)rank * 16 + c] = hyps[(size_t)i * 16 + c];
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------
// nr10: K10's rays per tile
static int launch_reloc_fused(Workspace& ws, const VmbLayout& L, const TrackParams& tp, const void* image,
                              const double* hyps, int n_hyp, double* scores, double* terms, int nr10, int n_sm,
                              cudaStream_t st, std::string& err) {
  if (L.H != 32 || L.nfreq != 6) { err = "relocalisation scoring: hidden must be 32 and n_freq 6"; return VMB_E_UNSUPPORTED; }
  if (tp.S < 1 || tp.S > 32) { err = "relocalisation scoring: n_samples must be in [1, 32]"; return VMB_E_UNSUPPORTED; }
  const int rpw = 32 / tp.S, nr = 4 * rpw;
  const int tiles = (tp.R + nr - 1) / nr;
  // chunks of hypotheses: enough CTAs for about four waves of two per SM, each CTA reusing its image and counts
  const long long ctas = (long long)tiles * tp.B;
  const int want = (int)std::max(1LL, std::min<long long>(n_hyp, (8LL * n_sm + ctas - 1) / ctas));
  const int chunk = (n_hyp + want - 1) / want, n_chunks = (n_hyp + chunk - 1) / chunk;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaError_t e = smem_limit_once<k_reloc_fused>(dev, tf::SMEM);
  if (e == cudaSuccess) e = ws.lray.grow((size_t)n_hyp * tp.B * tp.R * 3 * sizeof(double), stream_capturing(st));
  if (e != cudaSuccess) { err = std::string("relocalisation scoring: ") + cudaGetErrorString(e); return VMB_E_CUDA; }
  k_reloc_fused<<<dim3((unsigned)tiles, (unsigned)tp.B, (unsigned)n_chunks), NT, tf::SMEM, st>>>(
      tp, (const unsigned char*)image, hyps, n_hyp, chunk, nr, rpw, ws.lray);
  k_reloc_reduce<<<(unsigned)n_hyp, 256, 0, st>>>(tp.B, tp.R, nr10, (double)tp.cs, (double)tp.os, ws.lray, scores,
                                                  terms);
  e = cudaGetLastError();
  if (e != cudaSuccess) { err = std::string("relocalisation scoring launch: ") + cudaGetErrorString(e); return VMB_E_CUDA; }
  return 0;
}

}  // namespace rl
