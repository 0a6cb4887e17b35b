// K10 / K11 at hidden 32 on the tensor cores: the pose gradient of the vMAP object models through the wgmma tile of the
// fused training step (k_step_fused.cuh) instead of K10's fp32 CUDA cores.  One launch per group covers every object.
//
// The rule is K10's (k_track.cuh) and, for the BA flavour, K11's (k_ba.cuh): same samples, same points, same loss with
// the per-object, per-term empty-mask rule, same left-perturbation gradient, same output rows, so vmb_track_update and
// vmb_ba_update run unchanged on what this path writes.  The parts that do not depend on where the network runs are
// the helpers K10, K11 and the layer-wise path (k_track_lw.cuh) call too: ba_draw_frame, pose_point, ray_loss and
// pose_terms of k_track.cuh and slice_mask_count of k_step_fp32.cuh.  What differs is where the network runs and its
// precision:
//   Weights  object b reads the fp16 weight image row rows[b] ([n_rows][um::IMG_BYTES], as the AdamW launch writes it)
//            with one bulk async copy: the fp16 matrices, the fp32 biases and the PE directions.  rows[] stays a device
//            array (capturable); a row outside [0, n_rows) contributes zero rows and sets VMB_TRACK_ST_BAD_ROW, as K10.
//   Tile     uf::Tile, the fused step's (k_step_fused.cuh): one CTA = whole rays of one object (blockIdx.y), up to 128 points, 256 threads = two
//            warpgroups; rays never straddle a warp (32 / S rays per warp, S <= 32), so a tile is 4 (32 / S) rays.  Not
//            cooperative and no CTA waits on another: each CTA counts its object's mask slice in its prologue
//            (load_object, shared with k_reloc_fused).
//   Points   pose_point: p = R q + t from an fp32 copy of the fp64 pose, then p / scale.  K11: the pose of the ray's draw
//            frame (ba_draw_frame); a ray whose frame is outside the table contributes nothing and sets
//            VMB_BA_ST_BAD_FRAME.
//   Forward  forward_tile: uf::Tile::embed (E0) and the six forward wgmma stages (in_layer, mid1, cat_layer, mid2,
//            color_linear + out_alpha, out_color) with uf::Tile::epi_relu, the step's operand layout and fp16 rounding
//            points: fp16 embedding, fp16 image weights, fp32 accumulation, fp16 ReLU activations, fp32 heads.
//   Render   one lane per sample, the ray's lanes adjacent in a warp: the heads' sigmoids in fp32, then K10's render in
//            fp64 in sample order (1 - occ as sigmoid(-alpha)) and ray_loss on it, with the object's own mask counts.
//            Each ray's three loss terms stay in fp64.  d(raw alpha) and d(raw colour) in fp32 as K10, scaled by
//            um::LS = 2^8 and clamped to +-60000 before the fp16 pack into the dhead block.  status[1] gets a LOWER BOUND
//            on the clamped values (and VMB_TRACK_ST_CLAMP is set when it is not 0): exactly the dhead values (the
//            four per point: LS d(raw alpha), LS d(raw colour)[3]) whose magnitude passes 60000; the saturating fp16
//            packs of the d_hc .. d_fc1 epilogues are not counted.
//   Backward the fused step's input-gradient chain without its weight gradients: d_hc, d_fc4 (with the dhead . W_a
//            term), d_fc3, d_fc2, d_fc1, d_emb, each gated dY (uf::Tile::epi_dgrad) passed to the next wgmma in
//            registers, d_emb to the eg tile (uf::Tile::eg_store).  No dB, no partial rows of weights, no finish and no
//            AdamW.
//   Pose     per point dL/dt = INV_LS (dE_xyz + sum_d dproj_d B_d) from uf::Tile::pe_backward, the half sums the
//            fused step's JOINT instantiation stores (warpgroup 0: dE_xyz, directions 0..11; warpgroup 1: 12..20; the
//            two halves added in that order), then pose_terms ((R q) x g, g), g = dL/dt / scale, in fp64 from the fp64
//            pose.
//   Rows     one row per ray, its samples summed in sample order: K11's rows [B][R][VMB_TRACK_PART] (BA flavour).  The
//            track flavour writes the same per-ray terms to the workspace and k_tf_reduce sums them per K10 tile
//            (vmb_track_tiles' tile of 128 / S rays, which the fused tile matches only at S = 10 and 32) in ray order
//            by k_tlw_reduce's rule (tlw_reduce_row): K10's partial rows [B][vmb_track_tiles(32, R, S)][VMB_TRACK_PART].
// No floating-point atomics anywhere on this path: bitwise reproducible.  Integer status atomics only.
// Registers (ptxas -v, sm_90a), no spills in any of them: k_track_fused track / BA flavour 80 / 84; k_tf_reduce 40.
// Shared memory per CTA: 112,656 B dynamic (activations / embedding-gradient tile 80 KB, weight image 26 KB, heads tile,
// dL/dt halves, barrier) + 1 KB static, so two CTAs share an SM.
#pragma once
#include "k_step_fused.cuh"
#include "k_track_lw.cuh"

namespace tf {

constexpr int NT = 256, FGB = uf::FGB;
// feature blocks 0 .. 39 of the fused step's layout: DH, FC1, FC2, E1, FC3, FC4, E2, HC (no Z: no dY is stored, no
// dproj block: no dB).  The fp32 embedding-gradient tile aliases them: after d_fc1's epilogue nothing reads them.
constexpr int ACT_BYTES = (uf::FG_HC + 4) * FGB;
static_assert(uf::EG_BYTES <= ACT_BYTES, "the embedding-gradient tile fits over the activations");
constexpr int SM_ACT = 0, SM_W = ACT_BYTES, SM_HD = SM_W + um::IMG_BYTES, SM_DT = SM_HD + uf::HD_BYTES;
constexpr int DT_BYTES = 128 * 16;                    // warpgroup 1's half of dL/dt per point
constexpr int SM_BAR = SM_DT + DT_BYTES, SMEM = SM_BAR + 16;
constexpr float LS = um::LS, INV_LS = um::INV_LS;

// per-ray pose terms and loss terms of the track flavour (k_tf_reduce's input), handle scratch (DeviceBuffer's rule).
// Sized for the handle's max_obj objects (not the B of the call: the tracked set changes from frame to frame, and a
// frame that tracks more objects than the captured one must still run), so only a larger n_rays than any call before a
// capture is refused.
struct Workspace {
  DeviceBuffer<double> gray;   // [B][R][6]
  DeviceBuffer<double> lray;   // [B][R][3]
};

// The start of k_track_fused and k_reloc_fused once the object's image row is known to be valid: the weight image on
// its way behind the barrier at SM_BAR (image_ready waits for it) while the object's slice mask counts
// (loss.py:16-18,38) go to red -- every CTA of the object counts the same rays.  Returns the tile (quad: this thread's
// warp within its warpgroup); its embedding-gradient tile aliases the activations, which nothing reads after d_fc1.
__device__ __forceinline__ uf::Tile load_object(unsigned char* smem, const unsigned char* image, int row,
                                                const TrackParams& a, int (&red)[3][NT / 32], int quad) {
  const int tid = threadIdx.x, b = blockIdx.y, R = a.R;
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem + SM_BAR);
  if (tid == 0) { ptx::mbar_init(wbar, 1); ptx::mbar_init_fence(); }
  __syncthreads();
  if (tid == 0) {
    ptx::mbar_arrive_expect_tx(wbar, um::IMG_BYTES);
    ptx::bulk_g2s(smem + SM_W, image + (size_t)row * um::IMG_BYTES, um::IMG_BYTES, wbar);
  }
  const unsigned char* sv = a.sem + (size_t)b * a.sem_stride;
  const unsigned char* mv = a.mask + (size_t)b * a.mask_stride;
  int nd = 0, no = 0, ns = 0;
  for (int r = tid; r < R; r += NT) slice_mask_count(sv, mv, r, nd, no, ns);
  warp_mask_counts(tid, nd, no, ns, red);
  return uf::Tile(smem + SM_ACT, smem + SM_ACT, smem + SM_W, reinterpret_cast<float*>(smem + SM_HD), quad);
}

__device__ __forceinline__ void image_ready(unsigned char* smem) {
  um::mbar_wait_or_trap(reinterpret_cast<uint64_t*>(smem + SM_BAR), 0);
}

// E0 (uf::Tile::embed) and the six forward stages of one tile (the fused step's layout and fp16 rounding points) at this
// thread's network input: the embedding blocks and hidden activations to `act`, the heads (raw alpha, raw colour[3]) in
// point layout to `hd` and zeroed dhead rows.  The weight image is in shared memory.  Ends before the CTA barrier that makes
// the heads tile visible.  Shared by k_track_fused and the forward-only relocalisation tile (k_reloc.cuh).
__device__ __forceinline__ void forward_tile(const uf::Tile& tl, const uf::PeIn& in, uint32_t (&ua)[8]) {
  tl.embed(in);

#define MMA_DONE() do { ptx::wgmma_commit(); ptx::wgmma_wait<0>(); } while (0)

  // ---- forward: the fused step's six stages.  Only the embedding blocks cross warpgroups (SS A operand): one CTA
  // barrier; every later A operand is this warpgroup's own registers (RS) or the embedding blocks again -------------
  float acc[16], hacc[8];
  ptx::fence_async_smem();
  __syncthreads();
  ptx::wgmma_fence();                                 // in_layer: emb1 (K = 96)
#pragma unroll
  for (int ks = 0; ks < 6; ++ks) ptx::wgmma_n32<0, 0>(acc, tl.mm.a_k(uf::FG_E1, ks), tl.mm.w_k(um::IMG_WIN, ks), ks > 0);
  MMA_DONE();
  tl.epi_relu(acc, um::F_BIN, uf::FG_FC1, ua);
  ptx::wgmma_fence();                                 // mid1: fc1
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, tl.mm.w_k(um::IMG_WM1, ks), ks > 0);
  MMA_DONE();
  tl.epi_relu(acc, um::F_BM1, uf::FG_FC2, ua);
  ptx::wgmma_fence();                                 // cat_layer: [fc2 | emb1] (K = 128)
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, tl.mm.w_k(um::IMG_WCAT, ks), ks > 0);
#pragma unroll
  for (int ks = 2; ks < 8; ++ks) ptx::wgmma_n32<0, 0>(acc, tl.mm.a_k(uf::FG_FC2, ks), tl.mm.w_k(um::IMG_WCAT, ks), 1u);
  MMA_DONE();
  tl.epi_relu(acc, um::F_BCAT, uf::FG_FC3, ua);
  ptx::wgmma_fence();                                 // mid2: fc3
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, tl.mm.w_k(um::IMG_WM2, ks), ks > 0);
  MMA_DONE();
  tl.epi_relu(acc, um::F_BM2, uf::FG_FC4, ua);
  ptx::wgmma_fence();                                 // color_linear: [fc4 | emb2] (K = 80) ; out_alpha: fc4 -> column 0
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<0>(acc, ua + 4 * ks, tl.mm.w_k(um::IMG_WCL, ks), ks > 0);
#pragma unroll
  for (int ks = 2; ks < 5; ++ks) ptx::wgmma_n32<0, 0>(acc, tl.mm.a_k(uf::FG_FC4, ks), tl.mm.w_k(um::IMG_WCL, ks), 1u);
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16_rs<0>(hacc, ua + 4 * ks, tl.mm.w16_k(um::IMG_WA16, ks), ks > 0);
  MMA_DONE();
  tl.epi_relu(acc, um::F_BCL, uf::FG_HC, ua);
  if (tl.cq == 0) { tl.hd[tl.fr0 * 4] = hacc[0]; tl.hd[(tl.fr0 + 8) * 4] = hacc[2]; }
  ptx::wgmma_fence();                                 // out_color: hc -> columns 1..3
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16_rs<0>(hacc, ua + 4 * ks, tl.mm.w16_k(um::IMG_WOC16, ks), ks > 0);
  MMA_DONE();
  if (tl.cq == 0) { tl.hd[tl.fr0 * 4 + 1] = hacc[1]; tl.hd[(tl.fr0 + 8) * 4 + 1] = hacc[3]; }
  if (tl.cq == 1) { tl.hd[tl.fr0 * 4 + 2] = hacc[0]; tl.hd[tl.fr0 * 4 + 3] = hacc[1]; tl.hd[(tl.fr0 + 8) * 4 + 2] = hacc[2]; tl.hd[(tl.fr0 + 8) * 4 + 3] = hacc[3]; }
#undef MMA_DONE
}

// One sample's heads (point layout, from forward_tile) rendered along its ray by K10's rule, one lane per sample, the
// ray's lanes [seg_lo, seg_lo + S) adjacent in the warp (every lane of the ray runs the sums): the heads' sigmoids in
// fp32, then the fp64 render in sample order (1 - occ as sigmoid(-alpha)) and the detached depth variance.  Also this
// sample's transmittance and weight in fp32 (the backward's).
struct RayRender {
  float al, oc, c0, c1, c2, Ts, wgt;
  double D, O, C0, C1, C2, V;
};

__device__ __forceinline__ RayRender render_ray(const float* hd, const float* wf, float zv, int p, int S, int sidx,
                                                int seg_lo) {
  const unsigned FULL = 0xffffffffu;
  RayRender r;
  const float4 hv = *reinterpret_cast<const float4*>(hd + p * 4);
  const float al = (hv.x + wf[um::F_BA]) * 10.0f;  // model.py:77
  const float oc = vmb_sigmoid(al);                 // render_rays.py:6
  const float c0 = vmb_sigmoid(hv.y + wf[um::F_BOC]), c1 = vmb_sigmoid(hv.z + wf[um::F_BOC + 1]),
              c2 = vmb_sigmoid(hv.w + wf[um::F_BOC + 2]);
  double Tr = 1.0, D = 0.0, O = 0.0, C0 = 0.0, C1 = 0.0, C2 = 0.0;
  float Ts = 0.f, wgt = 0.f;
  for (int s = 0; s < S; ++s) {                     // the ray's samples in order
    const int src = seg_lo + s;
    const float al_s = __shfl_sync(FULL, al, src), oc_s = __shfl_sync(FULL, oc, src), z_s = __shfl_sync(FULL, zv, src);
    const float c0_s = __shfl_sync(FULL, c0, src), c1_s = __shfl_sync(FULL, c1, src), c2_s = __shfl_sync(FULL, c2, src);
    const double wd = (double)oc_s * Tr;
    if (sidx == s) { Ts = (float)Tr; wgt = (float)wd; }
    D += wd * (double)z_s; O += wd;
    C0 += wd * (double)c0_s; C1 += wd * (double)c1_s; C2 += wd * (double)c2_s;
    Tr *= ((double)vmb_sigmoid(-al_s) + 1e-10);
  }
  double V = 0.0;
  for (int s = 0; s < S; ++s) {
    const double dz = (double)__shfl_sync(FULL, zv, seg_lo + s) - D;
    V += (double)__shfl_sync(FULL, wgt, seg_lo + s) * dz * dz;   // loss.py:28-29 (detached)
  }
  r.al = al; r.oc = oc; r.c0 = c0; r.c1 = c1; r.c2 = c2; r.Ts = Ts; r.wgt = wgt;
  r.D = D; r.O = O; r.C0 = C0; r.C1 = C1; r.C2 = C2; r.V = V;
  return r;
}

// the object's slice mask counts (nd, no, ns) from warp_mask_counts' per-warp sums
__device__ __forceinline__ void red_counts(const int (&red)[3][NT / 32], int (&cnt)[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    cnt[c] = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) cnt[c] += red[c][w];
  }
}

// One CTA = tile blockIdx.x of object blockIdx.y.  nr = 4 rpw rays per tile, rpw = 32 / S rays per warp.
// BA = false: per-ray terms to gray / lray (k_tf_reduce forms K10's partials); BA = true: K11's rows x.rows.
template <bool BA>
__global__ void __launch_bounds__(NT, 2) k_track_fused(TrackParams a, BaRays x, const unsigned char* __restrict__ image,
                                                       int nr, int rpw, double* __restrict__ gray, double* __restrict__ lray) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ int red[3][NT / 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.y, S = a.S, R = a.R;
  const unsigned FULL = 0xffffffffu;
  // point layout (one thread pair per point) and this thread's sample; uf::Tile holds the fragment layout
  const int p = tid & 127, hsel = tid >> 7, quad = warp & 3;
  const int rw = lane / S, sidx = lane - rw * S, seg_lo = lane - sidx;
  const int ray = blockIdx.x * nr + quad * rpw + rw;
  const bool live = rw < rpw && ray < R;
  const size_t orow = (size_t)b * R + ray;            // this ray's output row
  const int row = a.rows[b];
  if (row < 0 || row >= a.n_rows) {                   // uniform over the CTA
    if (hsel == 0 && live && sidx == 0) {
      if constexpr (BA) {
        for (int c = 0; c < VMB_TRACK_PART; ++c) x.rows[orow * VMB_TRACK_PART + c] = 0.0;
      } else {
        for (int c = 0; c < 6; ++c) gray[orow * 6 + c] = 0.0;
        for (int c = 0; c < 3; ++c) lray[orow * 3 + c] = 0.0;
      }
    }
    if (tid == 0 && a.status) atomicOr(a.status, VMB_TRACK_ST_BAD_ROW);
    return;
  }
  const uf::Tile tl = load_object(smem, image, row, a, red, quad);

  // ---- points: p = R q + t (fp32 copy of the fp64 pose), network input p / scale ------------------------------------
  const double* T = a.pose;
  bool pok = live;                                    // K11: the ray's frame is in the pose table
  if constexpr (BA) {
    const int f = live ? ba_draw_frame(x.kf_draw, x.kf_draw_stride, x.kf_frame, x.kf_stride, x.n_poses, b, ray / x.n_pix_draw) : -1;
    pok = f >= 0;
    T = a.pose + (size_t)(pok ? f : 0) * 16;
  }
  const float sc = a.scale[row];
  float3 q = make_float3(0.f, 0.f, 0.f), t = q;
  if (pok) {
    const size_t gi = (size_t)b * a.pcs_stride + ((size_t)ray * S + sidx) * 3;
    q = make_float3(a.pcs[gi], a.pcs[gi + 1], a.pcs[gi + 2]);
    t = pose_point(T, q, sc);
  }
  float zv = 0.f;
  if (hsel == 0 && live) zv = a.z[(size_t)b * a.z_stride + (size_t)ray * S + sidx];

  image_ready(smem);

  const uf::PeIn tin(t);
  uint32_t ua[8];
  forward_tile(tl, tin, ua);
#define MMA_DONE() do { ptx::wgmma_commit(); ptx::wgmma_wait<0>(); } while (0)
  float acc[16], hacc[8];
  __syncthreads();                                    // heads tile (fragment layout -> point layout); mask counts

  // ---- render + loss + d(raw alpha, raw colour): K10's rule, one lane per sample in the warps of warpgroup 0 ---------
  if (hsel == 0) {                                    // warp-uniform
    const RayRender rr = render_ray(tl.hd, tl.wf, zv, p, S, sidx, seg_lo);
    const float al = rr.al, oc = rr.oc, c0 = rr.c0, c1 = rr.c1, c2 = rr.c2, Ts = rr.Ts, wgt = rr.wgt;
    const double D = rr.D, O = rr.O, C0 = rr.C0, C1 = rr.C1, C2 = rr.C2, V = rr.V;
    int cnt[3];
    red_counts(red, cnt);
    RayLoss ls = {{0.0, 0.0, 0.0}, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (live) {
      if (BA && !pok && sidx == 0 && a.status) atomicOr(a.status, VMB_BA_ST_BAD_FRAME);
      ls = ray_loss(D, O, C0, C1, C2, V, a.sem[(size_t)b * a.sem_stride + ray], a.mask[(size_t)b * a.mask_stride + ray] != 0,
                    a.gt_depth[(size_t)b * a.gt_depth_stride + ray], a.gt_colour + (size_t)b * a.gt_colour_stride + (size_t)ray * 3,
                    pok, cnt, a.cs, a.os);
      if (sidx == 0) {
        if constexpr (BA) {
          double* o = x.rows + orow * VMB_TRACK_PART;
          o[6] = ls.l[0]; o[7] = ls.l[1]; o[8] = ls.l[2]; o[9] = 0.0;
        } else {
          lray[orow * 3] = ls.l[0]; lray[orow * 3 + 1] = ls.l[1]; lray[orow * 3 + 2] = ls.l[2];
        }
      }
    }
    const float Gs = fmaf(ls.gD, zv, fmaf(ls.gC0, c0, fmaf(ls.gC1, c1, fmaf(ls.gC2, c2, ls.gO))));
    const float fr = vmb_sigmoid(-al);                // 1 - occ
    float suffix = 0.f, docc = 0.f;                   // K10's suffix sum, samples from the last
    for (int s = S - 1; s >= 0; --s) {
      if (sidx == s) docc = Gs * Ts - suffix / (fr + 1e-10f);
      suffix = fmaf(__shfl_sync(FULL, Gs, seg_lo + s), __shfl_sync(FULL, wgt, seg_lo + s), suffix);
    }
    int n_clamp = 0;
    if (live) {
      float d[4] = {LS * (10.0f * docc * oc * fr), LS * (ls.gC0 * wgt * c0 * (1.f - c0)), LS * (ls.gC1 * wgt * c1 * (1.f - c1)),
                    LS * (ls.gC2 * wgt * c2 * (1.f - c2))};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        n_clamp += fabsf(d[c]) > 60000.f;
        d[c] = fminf(fmaxf(d[c], -60000.f), 60000.f);
      }
      *reinterpret_cast<uint2*>(tl.act + uf::FG_DH * FGB + p * 16) = make_uint2(um::pack_h2(d[0], d[1]), um::pack_h2(d[2], d[3]));
    }
    for (int o = 16; o > 0; o >>= 1) n_clamp += __shfl_xor_sync(FULL, n_clamp, o);
    if (lane == 0 && n_clamp && a.status) { atomicOr(a.status, VMB_TRACK_ST_CLAMP); atomicAdd(a.status + 1, n_clamp); }
  }

  // ---- backward to the embedding only: dhead (point layout, SS) crosses warpgroups, then every A is registers --------
  uint32_t uyc[8], uy3[8];
  ptx::fence_async_smem();
  __syncthreads();
  ptx::wgmma_fence();                                 // d_hc = dhead @ W_oc
  ptx::wgmma_n32<0, 1>(acc, tl.mm.a_k(uf::FG_DH, 0), tl.mm.w16_mn(um::IMG_WOC16), 0u);
  MMA_DONE();
  tl.epi_dgrad<false>(acc, uf::FG_HC, 0, uyc);
  ptx::wgmma_fence();                                 // d_fc4 = dYc @ W_cl[:, :32] + dhead @ W_a
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uyc + 4 * ks, tl.mm.w_mn(um::IMG_WCL, ks), ks > 0);
  ptx::wgmma_n32<0, 1>(acc, tl.mm.a_k(uf::FG_DH, 0), tl.mm.w16_mn(um::IMG_WA16), 1u);
  MMA_DONE();
  tl.epi_dgrad<false>(acc, uf::FG_FC4, 0, ua);
  ptx::wgmma_fence();                                 // d_fc3 = dY4 @ W_m2
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, ua + 4 * ks, tl.mm.w_mn(um::IMG_WM2, ks), ks > 0);
  MMA_DONE();
  tl.epi_dgrad<false>(acc, uf::FG_FC3, 0, uy3);
  ptx::wgmma_fence();                                 // d_fc2 = dY3 @ W_cat[:, :32]
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uy3 + 4 * ks, tl.mm.w_mn(um::IMG_WCAT, ks), ks > 0);
  MMA_DONE();
  tl.epi_dgrad<false>(acc, uf::FG_FC2, 0, ua);
  ptx::wgmma_fence();                                 // d_fc1 = dY2 @ W_m1
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, ua + 4 * ks, tl.mm.w_mn(um::IMG_WM1, ks), ks > 0);
  MMA_DONE();
  tl.epi_dgrad<false>(acc, uf::FG_FC1, 0, ua);
  __syncthreads();                                    // every read of the activations is done: eg may overwrite them
  // d_emb1 = dY3 @ W_cat[:, 32:] + dY1 @ W_in (32 columns at a time), d_emb2 = dYc @ W_cl[:, 32:]
  ptx::wgmma_fence();
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uy3 + 4 * ks, tl.mm.w_mn(um::IMG_WCAT + (4 + 4 * c) * 512, ks), ks > 0);
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, ua + 4 * ks, tl.mm.w_mn(um::IMG_WIN + 4 * c * 512, ks), 1u);
    MMA_DONE();
    tl.eg_store(acc, 8 * c);
    ptx::wgmma_fence();
  }
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n32_rs<1>(acc, uyc + 4 * ks, tl.mm.w_mn(um::IMG_WCL + 4 * 512, ks), ks > 0);
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) ptx::wgmma_n16_rs<1>(hacc, uyc + 4 * ks, tl.mm.w_mn(um::IMG_WCL + 8 * 512, ks), ks > 0);
  MMA_DONE();
  tl.eg_store(acc, uf::EG_E2);
  tl.eg_store(hacc, uf::EG_E2 + 8);
#undef MMA_DONE
  __syncthreads();                                    // embedding-gradient tile: fragment layout -> point layout

  // ---- PE backward: this warpgroup's half of dL/dt, warpgroup 1's to shared memory ------------------------------------
  const float3 jt = tl.pe_backward<false>(tin);
  if (hsel) *reinterpret_cast<float4*>(smem + SM_DT + p * 16) = make_float4(jt.x, jt.y, jt.z, 0.f);
  __syncthreads();

  // ---- pose terms in fp64 per point, the ray's samples summed in order into its row ---------------------------------
  if (hsel == 0) {
    const float4 h1 = *reinterpret_cast<const float4*>(smem + SM_DT + p * 16);
    double c6[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (pok) pose_terms(T, make_double3(q.x, q.y, q.z), make_float3(jt.x + h1.x, jt.y + h1.y, jt.z + h1.z), sc, c6);
    double s6[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int s = 0; s < S; ++s)
#pragma unroll
      for (int c = 0; c < 6; ++c) s6[c] += __shfl_sync(FULL, c6[c], seg_lo + s);
    if (live && sidx == 0) {
      double* o = BA ? x.rows + orow * VMB_TRACK_PART : gray + orow * 6;
#pragma unroll
      for (int c = 0; c < 6; ++c) o[c] = s6[c];
    }
  }
}

// K10's partial rows of the track flavour: row j of object blockIdx.y sums the per-ray terms of rays
// [j nr10, (j + 1) nr10) in ray order (k_tlw_reduce's rule, one "point" per ray), nr10 = K10's rays per tile
__global__ void __launch_bounds__(128) k_tf_reduce(int R, int nr10, int n_out, const double* __restrict__ gray,
                                                   const double* __restrict__ lray, double* __restrict__ partials) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_out) return;
  const size_t b = blockIdx.y;
  lw::tlw_reduce_row(R, 1, nr10, j, true, gray + b * R * 6, lray + b * R * 3, partials + (b * n_out + j) * VMB_TRACK_PART);
}

// ---------------------------------------------------------------------------------------------------------------------
// host: one launch for every object of the group (+ k_tf_reduce for the track flavour)
// ---------------------------------------------------------------------------------------------------------------------
// cap_obj: the handle's max_obj, the object count the track flavour's workspace is sized for (B, if larger)
template <bool BA>
static int launch_track_fused(Workspace& ws, const VmbLayout& L, const TrackParams& tp, const BaRays& x, const void* image,
                              int nr10, int cap_obj, cudaStream_t st, std::string& err) {
  if (L.H != 32 || L.nfreq != 6) { err = "fused tracking step: hidden must be 32 and n_freq 6"; return VMB_E_UNSUPPORTED; }
  if (tp.S < 1 || tp.S > 32) { err = "fused tracking step: n_samples must be in [1, 32]"; return VMB_E_UNSUPPORTED; }
  const int rpw = 32 / tp.S, nr = 4 * rpw;
  const int tiles = (tp.R + nr - 1) / nr;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaError_t e = smem_limit_once<k_track_fused<BA>>(dev, SMEM);
  if (e == cudaSuccess && !BA) {
    const size_t rays = (size_t)std::max(cap_obj, tp.B) * tp.R;
    const bool capturing = stream_capturing(st);
    e = ws.gray.grow(rays * 6 * sizeof(double), capturing);
    if (e == cudaSuccess) e = ws.lray.grow(rays * 3 * sizeof(double), capturing);
  }
  if (e != cudaSuccess) { err = std::string("fused tracking step: ") + cudaGetErrorString(e); return VMB_E_CUDA; }
  k_track_fused<BA><<<dim3((unsigned)tiles, (unsigned)tp.B), NT, SMEM, st>>>(tp, x, (const unsigned char*)image, nr, rpw,
                                                                            ws.gray, ws.lray);
  if (!BA) {
    const int n_out = (tp.R + nr10 - 1) / nr10;
    k_tf_reduce<<<dim3((unsigned)((n_out + 127) / 128), (unsigned)tp.B), 128, 0, st>>>(tp.R, nr10, n_out, ws.gray, ws.lray,
                                                                                      tp.partials);
  }
  e = cudaGetLastError();
  if (e != cudaSuccess) { err = std::string("fused tracking step launch: ") + cudaGetErrorString(e); return VMB_E_CUDA; }
  return 0;
}

}  // namespace tf
