// K10 / K11 on the layer-wise tensor-core path: the pose gradient of a wide model (hidden 64 / 128 / 256: the iMAP
// whole-scene model, the vMAP background) through the wgmma GEMMs of k_layerwise.cuh instead of K10's fp32 CUDA cores.
//
// The rule is K10's (k_track.cuh) and, for the BA flavour, K11's (k_ba.cuh): same samples, same points, same loss with
// the per-object, per-term empty-mask rule, same left-perturbation gradient, same output rows, so vmb_track_update and
// vmb_ba_update run unchanged on what this path writes.  The parts that do not depend on where the network runs are
// the helpers that K10 and K11 call too: ba_draw_frame, pose_point, ray_loss and pose_terms of k_track.cuh and
// slice_mask_count of k_step_fp32.cuh.  What differs is where the network runs and its precision:
//   Weights  object b reads params row rows[b] and the fp16 image row rows[b] (as the AdamW launch writes it).  Both
//            are copied on the device into this path's workspace first, so rows[] stays a device array (capturable);
//            a row outside [0, n_rows) contributes nothing and sets VMB_TRACK_ST_BAD_ROW, as K10.
//   Points   pose_point: p = R q + t from an fp32 copy of the fp64 pose, then p / scale; the embedding block is
//            k_lw_pe's pe_block (fp16, sin by sincos_ladder6, constant-1 columns).  K11: the ray's pose is its draw's
//            frame (ba_draw_frame); a ray whose frame is outside the table contributes nothing and sets
//            VMB_BA_ST_BAD_FRAME.
//   Network  the five forward GEMMs of step_object (fp16 operands, fp32 accumulation, fp16 activations).
//   Render   one warp per ray, lane = sample (S <= 32): the training kernel's HeadRows (row staging, the heads in fp32
//            from the fp16 activations, the dYc gate and its store); the composite, render in fp64 in sample order
//            exactly as K10 (1 - occ as sigmoid(-alpha)) and ray_loss on it; mask counts of this slice per object
//            (integers); the backward to (raw alpha, raw colour) in fp32 as K10.  Each ray's three loss terms go to an
//            fp64 per-ray buffer.  d(raw alpha) and dYc are loss-scaled by LS = 2^8 and clamped to the fp16 range
//            +-60000 as in the training kernel.  status[1] gets a LOWER BOUND on the clamped values (and
//            VMB_TRACK_ST_CLAMP is set when it is not 0), the count HeadRows::gate returns: every clamped dYc element,
//            plus every element where the rank-1 term LS d(raw alpha) W_a of dY4 passes 60000 on its own; the
//            saturating packs of the dY4..dY1 GEMM epilogues are not counted.  No head weight gradients.
//   Backward step_object's input-gradient chain (InputGrads: colour-block dE, dY4 with the rank-1 d_alpha term, dY3,
//            dY2, dY1, the fused dE GEMM) back to back: no weight-gradient GEMMs, no column sums, no side stream.
//   Pose     per point dL/dt = INV_LS (dE_xyz + sum_{k,d} dE_{k,d} pi 2^k cos(pi 2^k proj_d) B_d) in fp32 (the cosines
//            of sincos_ladder6, as k_lw_pe_bwd), then pose_terms: ((R q) x g, g), g = dL/dt / scale, in fp64 from the
//            fp64 pose.  Track flavour: the terms are summed in point order over the rays of each of K10's tiles
//            (nr = TP / S rays, TP = vmb_track_tiles' tile), plus the per-ray loss terms in ray order: exactly K10's
//            partial rows.  BA flavour: one row per ray (its samples in order), as K11.
// No floating-point atomics anywhere on this path (the GEMM epilogues used here store): bitwise reproducible.
// Registers (ptxas -v, sm_90a; track / BA flavour), no spills in any of them:
//   k_tlw_gather 32; k_tlw_pe 74 / 74; k_tlw_render 67 / 68 at every H; k_tlw_pose 62 / 62; k_tlw_reduce 40 / 40;
//   the joint step's k_joint_world 32 (it runs k_tlw_pose / k_tlw_reduce<true>).  The training step's kernels on the
//   same helpers: k_lw_pe 74, k_lw_heads_render 62 / 62 / 61 at H 64 / 128 / 256 (it drops HeadRows::gate's count).
#pragma once
#include "k_layerwise.cuh"
#include "k_track.cuh"

namespace lw {

// the path's own buffers next to the training step's (handle scratch, DeviceBuffer's rule)
struct TrackWorkspace {
  Workspace w;                          // E, X1..X4, XC, dYa..dYc, dalpha_s, dE (dh16 unused)
  DeviceBuffer<float> prow;             // [stride] the object's fp32 param row
  DeviceBuffer<__half> wimg;            // [img_halves] its fp16 image row
  DeviceBuffer<int> ctl;                // [8]: mask counts nd, no, ns; row ok; scale (float bits)
  DeviceBuffer<double> lossr;           // [R][3] per-ray loss terms
  DeviceBuffer<double> gpt;             // [P][6] per-point pose terms
};

// What the path reads for one object b of the group (TrackParams / BaRays of k_track.cuh carry the rest)
struct TlwObj {
  int b, R, S, n_rows, n_pix_draw, n_poses, kf_stride;
  const int* rows;
  const float* pcs;                  // object b's slice [R][S][3]
  const double* pose;                // track: [16]; BA: the table [n_poses][16]
  const int* kf_draw; const int* kf_frame;   // BA: object b's rows
  int* status;
};

// frame id of ray r (BA) or 0 (track); -1 = outside the pose table
template <bool BA>
__device__ __forceinline__ int tlw_frame(const TlwObj& o, int r) {
  return BA ? ba_draw_frame(o.kf_draw, 0, o.kf_frame, o.kf_stride, o.n_poses, 0, r / o.n_pix_draw) : 0;
}

// ---- 1: the object's weights into the workspace; block 0 also counts the slice's masks (loss.py:16-18,38) ----------
__global__ void __launch_bounds__(256) k_tlw_gather(TlwObj o, const float* __restrict__ params, const float* __restrict__ scale,
                                                    const __half* __restrict__ image, const unsigned char* __restrict__ sem,
                                                    const unsigned char* __restrict__ mask, int stride, long long halves,
                                                    float* __restrict__ prow, __half* __restrict__ wimg, int* __restrict__ ctl) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const int row = o.rows[o.b];
  const bool ok = row >= 0 && row < o.n_rows;
  const long long n4 = halves / 8;                    // image rows are whole multiples of 16 B
  const uint4* src = reinterpret_cast<const uint4*>(image + (size_t)(ok ? row : 0) * halves);
  uint4* dst = reinterpret_cast<uint4*>(wimg);
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  for (long long i = t0; i < n4; i += nt) dst[i] = ok ? src[i] : make_uint4(0u, 0u, 0u, 0u);
  const float* P = params + (size_t)(ok ? row : 0) * stride;
  for (long long i = t0; i < stride; i += nt) prow[i] = ok ? P[i] : 0.f;
  if (blockIdx.x != 0) return;
  __shared__ int s_cnt[3];
  if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  int nd = 0, no = 0, ns = 0;
  for (int r = threadIdx.x; r < o.R; r += blockDim.x) slice_mask_count(sem, mask, r, nd, no, ns);
  atomicAdd(&s_cnt[0], nd); atomicAdd(&s_cnt[1], no); atomicAdd(&s_cnt[2], ns);
  __syncthreads();
  if (threadIdx.x < 3) ctl[threadIdx.x] = s_cnt[threadIdx.x];
  if (threadIdx.x == 3) ctl[3] = ok ? 1 : 0;
  if (threadIdx.x == 4) ctl[4] = __float_as_int(ok ? scale[row] : 1.0f);
  if (threadIdx.x == 5 && !ok && o.status) atomicOr(o.status, VMB_TRACK_ST_BAD_ROW);
}

// camera-frame point q and network input t = pose_point(q) of point p = ray r, sample s; false where the ray has no pose
template <bool BA>
__device__ __forceinline__ bool tlw_point(const TlwObj& o, long long p, float sc, float3& q, float3& t, const double*& T) {
  const int f = tlw_frame<BA>(o, (int)(p / o.S));
  q = t = make_float3(0.f, 0.f, 0.f);
  T = o.pose + (size_t)(f > 0 ? f : 0) * 16;
  if (f < 0) return false;
  q = make_float3(o.pcs[p * 3], o.pcs[p * 3 + 1], o.pcs[p * 3 + 2]);
  t = pose_point(T, q, sc);
  return true;
}

// ---- 2: positional embedding at the pose, k_lw_pe's row layout ------------------------------------------------------
template <bool BA>
__global__ void __launch_bounds__(128) k_tlw_pe(TlwObj o, const float* __restrict__ prow, const int* __restrict__ ctl, int o_B,
                                                __half* __restrict__ E) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const long long P = (long long)o.R * o.S;
  const float sc = __int_as_float(ctl[4]);
  const long long p = (long long)blockIdx.x * 128 + threadIdx.x;
  float3 q, t = make_float3(0.f, 0.f, 0.f);
  const double* T;
  if (p < P) tlw_point<BA>(o, p, sc, q, t, T);
  pe_block(t.x, t.y, t.z, prow + o_B, P, E);
}

// ---- 3: heads + fp64 render + loss + d(raw alpha, raw colour) -> dalpha_s, dYc; one warp per ray, lane = sample ------
struct TlwRender {
  const float* z; const float* gt_depth; const float* gt_colour; const unsigned char* sem; const unsigned char* mask;
  float cs, os;
};
template <int H, bool BA>
__global__ void __launch_bounds__(128) k_tlw_render(TlwObj o, TlwRender a, const __half* __restrict__ X4, const __half* __restrict__ XC,
                                                    const float* __restrict__ P, VmbLayout L, const int* __restrict__ ctl,
                                                    __half* __restrict__ dYc, float* __restrict__ dalpha_s, double* __restrict__ lossr) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  extern __shared__ __align__(16) unsigned char hr_rows[];
  __shared__ float w[4 * H];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, S = o.S;
  HeadRows<H> hr{w, hr_rows + warp * (32 * HeadRows<H>::PITCH), lane, S};
  hr.load(P, L);
  __syncthreads();
  const unsigned FULL = 0xffffffffu;
  const float b_a = P[L.o_ba], b_c0 = P[L.o_boc], b_c1 = P[L.o_boc + 1], b_c2 = P[L.o_boc + 2];
  const int cnt[3] = {ctl[0], ctl[1], ctl[2]};
  const bool in = lane < S;
  int n_clamp = 0;
  for (int ray = blockIdx.x * 4 + warp; ray < o.R; ray += gridDim.x * 4) {
    const long long pb = (long long)ray * S, pi = pb + lane;
    hr.stage(X4, pb);
    float ha = 0.f, h0 = 0.f, h1 = 0.f, h2 = 0.f;
    if (in) ha = hr.alpha();
    hr.stage(XC, pb);
    float al = 0.f, oc = 0.f, zz = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
    if (in) {
      hr.colour(h0, h1, h2);
      al = (ha + b_a) * 10.0f;                        // model.py:77
      oc = vmb_sigmoid(al);                           // render_rays.py:6
      c0 = vmb_sigmoid(h0 + b_c0); c1 = vmb_sigmoid(h1 + b_c1); c2 = vmb_sigmoid(h2 + b_c2);
      zz = a.z[pi];
    }
    // K10's per-ray render in fp64, samples in order (every lane runs the same sums)
    double Tr = 1.0, D = 0.0, O = 0.0, C0 = 0.0, C1 = 0.0, C2 = 0.0;
    float Ts = 0.f, wf = 0.f;
    for (int s = 0; s < S; ++s) {
      const float al_s = __shfl_sync(FULL, al, s), oc_s = __shfl_sync(FULL, oc, s), z_s = __shfl_sync(FULL, zz, s);
      const float c0_s = __shfl_sync(FULL, c0, s), c1_s = __shfl_sync(FULL, c1, s), c2_s = __shfl_sync(FULL, c2, s);
      const double wd = (double)oc_s * Tr;
      if (lane == s) { Ts = (float)Tr; wf = (float)wd; }
      D += wd * (double)z_s; O += wd;
      C0 += wd * (double)c0_s; C1 += wd * (double)c1_s; C2 += wd * (double)c2_s;
      Tr *= ((double)vmb_sigmoid(-al_s) + 1e-10);
    }
    double V = 0.0;
    for (int s = 0; s < S; ++s) {
      const double dz = (double)__shfl_sync(FULL, zz, s) - D;
      V += (double)__shfl_sync(FULL, wf, s) * dz * dz;  // loss.py:28-29 (detached)
    }
    const bool rok = tlw_frame<BA>(o, ray) >= 0;
    if (BA && !rok && lane == 0 && o.status) atomicOr(o.status, VMB_BA_ST_BAD_FRAME);
    const RayLoss ls = ray_loss(D, O, C0, C1, C2, V, a.sem[ray], a.mask[ray] != 0, a.gt_depth[ray], a.gt_colour + (size_t)ray * 3,
                                rok, cnt, a.cs, a.os);
    if (lane == 0)
      for (int c = 0; c < 3; ++c) lossr[(size_t)ray * 3 + c] = ls.l[c];
    const float gD = ls.gD, gC0 = ls.gC0, gC1 = ls.gC1, gC2 = ls.gC2, gO = ls.gO;
    const float Gs = fmaf(gD, zz, fmaf(gC0, c0, fmaf(gC1, c1, fmaf(gC2, c2, gO))));
    const float fr = vmb_sigmoid(-al);               // 1 - occ
    float suffix = 0.f, docc = 0.f;                   // K10's suffix sum, samples from the last
    for (int s = S - 1; s >= 0; --s) {
      if (lane == s) docc = Gs * Ts - suffix / (fr + 1e-10f);
      suffix = fmaf(__shfl_sync(FULL, Gs, s), __shfl_sync(FULL, wf, s), suffix);
    }
    if (in) {
      const float dx = 10.0f * docc * oc * fr;
      const float dy0 = gC0 * wf * c0 * (1.f - c0), dy1 = gC1 * wf * c1 * (1.f - c1), dy2 = gC2 * wf * c2 * (1.f - c2);
      const float da = LS * dx;
      dalpha_s[pi] = da;
      n_clamp += hr.gate(LS * dy0, LS * dy1, LS * dy2, da);
    }
    hr.store(dYc, pb);
  }
  for (int d = 16; d > 0; d >>= 1) n_clamp += __shfl_xor_sync(FULL, n_clamp, d);
  if (lane == 0 && n_clamp && o.status) { atomicOr(o.status, VMB_TRACK_ST_CLAMP); atomicAdd(o.status + 1, n_clamp); }
}

// ---- 4: per-point pose terms ((R q) x g, g) in fp64 ------------------------------------------------------------------
template <bool BA>
__global__ void __launch_bounds__(128) k_tlw_pose(TlwObj o, const float* __restrict__ prow, const int* __restrict__ ctl, int o_B,
                                                  const float* __restrict__ dE, double* __restrict__ gpt) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  extern __shared__ float sg[];                       // [128 points][PEB_LD]
  const long long P = (long long)o.R * o.S;
  const long long p0 = (long long)blockIdx.x * 128, p = p0 + threadIdx.x;
  stage_de_rows(sg, dE, p0, P);
  __syncthreads();
  if (p >= P) return;
  const float sc = __int_as_float(ctl[4]);
  const float* dirs = prow + o_B;
  float3 q, t;
  const double* T;
  const bool pok = tlw_point<BA>(o, p, sc, q, t, T);
  const float* g = sg + threadIdx.x * PEB_LD;
  float dt0 = g[0] * INV_LS, dt1 = g[1] * INV_LS, dt2 = g[2] * INV_LS;
#pragma unroll 1
  for (int d = 0; d < VMB_NDIRS; ++d) {
    const float b0 = dirs[d * 3], b1 = dirs[d * 3 + 1], b2 = dirs[d * 3 + 2];
    float s[6], c[6];
    sincos_ladder6(fmaf(b2, t.z, fmaf(b1, t.y, b0 * t.x)), s, c);
    const float dp = pe_dproj(g, d, c) * (VMB_PI_F * INV_LS);       // as k_lw_pe_bwd
    dt0 = fmaf(dp, b0, dt0); dt1 = fmaf(dp, b1, dt1); dt2 = fmaf(dp, b2, dt2);
  }
  double c6[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (pok && ctl[3]) pose_terms(T, make_double3(q.x, q.y, q.z), make_float3(dt0, dt1, dt2), sc, c6);
#pragma unroll
  for (int i = 0; i < 6; ++i) gpt[p * 6 + i] = c6[i];
}

// ---- 5: fixed-order fp64 sums into K10's partial rows (track) or K11's per-ray rows (BA) -----------------------------
// Row j of R rays of S points: the points' terms of rays [j per, (j + 1) per) in point order, their loss terms in ray
// order (0 when !ok, loss columns 0 when lossr is NULL).  Also the rule of the fused path's k_tf_reduce (S = 1).
__device__ __forceinline__ void tlw_reduce_row(int R, int S, int per, int j, bool ok, const double* __restrict__ gpt,
                                               const double* __restrict__ lossr, double* __restrict__ dst) {
  const int r0 = j * per, r1 = min(R, r0 + per);
  double s[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (ok) {
    const long long pe = (long long)r1 * S;
    for (long long p = (long long)r0 * S; p < pe; ++p)
#pragma unroll
      for (int c = 0; c < 6; ++c) s[c] += gpt[p * 6 + c];
    if (lossr)
      for (int r = r0; r < r1; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) s[6 + c] += lossr[(size_t)r * 3 + c];
  }
#pragma unroll
  for (int c = 0; c < 9; ++c) dst[c] = s[c];
  dst[9] = 0.0;
}

// lossr NULL (the joint step): the loss columns are written as 0
template <bool BA>
__global__ void __launch_bounds__(128) k_tlw_reduce(TlwObj o, int nr, int n_out, const int* __restrict__ ctl,
                                                    const double* __restrict__ gpt, const double* __restrict__ lossr,
                                                    double* __restrict__ out) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_out) return;
  tlw_reduce_row(o.R, o.S, BA ? 1 : nr, j, ctl[3] != 0, gpt, lossr, out + (size_t)j * VMB_TRACK_PART);
}

// ---------------------------------------------------------------------------------------------------------------------
// host: one object at a time on `st`
// ---------------------------------------------------------------------------------------------------------------------
struct TlwGroup {
  TrackParams tp;                // K10's group arguments (partials: track flavour output)
  BaRays x;                      // K11's (BA flavour: rows = output, kf_* the draw tables)
  const __half* image;           // [n_rows][img_halves(H)]
  int nr;                        // track flavour: rays per K10 tile
};

template <int H, bool BA>
static int track_object_lw(TrackWorkspace& tw, const VmbLayout& L, const TlwGroup& G, int b, cudaStream_t st, std::string& err) {
  const TrackParams& a = G.tp;
  Workspace& ws = tw.w;
  const long long np = (long long)a.R * a.S;
  const int nblk = (int)((np + 127) / 128);
  auto arm = [&]() { if (pdl_ok(np)) pdl_arm(); };
  TlwObj o;
  o.b = b; o.R = a.R; o.S = a.S; o.n_rows = a.n_rows; o.rows = a.rows;
  o.pcs = a.pcs + (size_t)b * a.pcs_stride; o.pose = a.pose; o.status = a.status;
  o.n_pix_draw = BA ? G.x.n_pix_draw : 1; o.n_poses = BA ? G.x.n_poses : 1; o.kf_stride = BA ? G.x.kf_stride : 0;
  o.kf_draw = BA ? G.x.kf_draw + (size_t)b * G.x.kf_draw_stride : nullptr;
  o.kf_frame = BA ? G.x.kf_frame + (size_t)b * G.x.kf_stride : nullptr;
  const unsigned char* sem = a.sem + (size_t)b * a.sem_stride;
  const unsigned char* mask = a.mask + (size_t)b * a.mask_stride;
  const long long halves = img_halves(H);
  int dev = 0;
  cudaGetDevice(&dev);
  const int n_sm = sm_count(dev);
  LW_TRY(launch_k(k_tlw_gather, dim3((unsigned)std::min<long long>(2 * n_sm, (halves / 8 + 255) / 256)), dim3(256), 0, st, o,
                  a.params, a.scale, G.image, sem, mask, L.stride, halves, tw.prow, tw.wimg, tw.ctl));
  arm();
  LW_TRY(launch_k(k_tlw_pe<BA>, dim3(nblk), dim3(128), 0, st, o, (const float*)tw.prow, (const int*)tw.ctl, L.o_B, ws.E));
  LW_TRY(forward_gemms<H>(ws, L, tw.prow, tw.wimg, np, st));
  LW_TRY((smem_limit_once<k_tlw_render<H, BA>>(dev, hr_smem<H>())));
  TlwRender ra;
  ra.z = a.z + (size_t)b * a.z_stride; ra.gt_depth = a.gt_depth + (size_t)b * a.gt_depth_stride;
  ra.gt_colour = a.gt_colour + (size_t)b * a.gt_colour_stride; ra.sem = sem; ra.mask = mask; ra.cs = a.cs; ra.os = a.os;
  arm();
  LW_TRY(launch_k(k_tlw_render<H, BA>, dim3(hr_blocks<H>(a.R, n_sm)), dim3(128), (size_t)hr_smem<H>(), st,
                  o, ra, (const __half*)ws.X4, (const __half*)ws.XC, (const float*)tw.prow, L, (const int*)tw.ctl, ws.dYc,
                  ws.dalpha_s, tw.lossr));
  // backward to the embedding only: step_object's input-gradient chain, each GEMM following the last directly
  const InputGrads<H> ig{ws, tw.wimg, tw.prow + L.o_Wa, np, st};
  arm();
  LW_TRY(ig.de_colour());
  arm();
  LW_TRY(ig.dy4());
  arm();
  LW_TRY(ig.dy3());
  arm();
  LW_TRY(ig.dy2());
  arm();
  LW_TRY(ig.dy1());
  arm();
  LW_TRY(ig.demb1());
  LW_TRY(smem_limit_once<k_tlw_pose<BA>>(dev, PEB_SMEM));
  arm();
  LW_TRY(launch_k(k_tlw_pose<BA>, dim3(nblk), dim3(128), (size_t)PEB_SMEM, st, o, (const float*)tw.prow, (const int*)tw.ctl, L.o_B,
                   (const float*)ws.dE, tw.gpt));
  const int n_out = BA ? a.R : (a.R + G.nr - 1) / G.nr;
  double* out = BA ? G.x.rows + (size_t)b * a.R * VMB_TRACK_PART : a.partials + (size_t)b * n_out * VMB_TRACK_PART;
  arm();
  LW_TRY(launch_k(k_tlw_reduce<BA>, dim3((n_out + 127) / 128), dim3(128), 0, st, o, G.nr, n_out, (const int*)tw.ctl,
                  (const double*)tw.gpt, (const double*)tw.lossr, out));
  LW_TRY(cudaGetLastError());
  return 0;
}

template <bool BA>
static int launch_track_lw(TrackWorkspace& tw, const VmbLayout& L, const TlwGroup& G, cudaStream_t st, std::string& err) {
  return for_hidden(L.H, "layer-wise tracking", err, [&](auto h) -> int {
    const long long R = G.tp.R, P = R * G.tp.S;
    const bool capturing = stream_capturing(st);
    LW_TRY(tw.w.grow(P, L.H, capturing));
    LW_TRY(tw.prow.grow((size_t)L.stride * 4, capturing));
    LW_TRY(tw.wimg.grow((size_t)img_halves(L.H) * 2, capturing));
    LW_TRY(tw.ctl.grow(8 * sizeof(int), capturing));
    LW_TRY(tw.lossr.grow((size_t)R * 3 * sizeof(double), capturing));
    LW_TRY(tw.gpt.grow((size_t)pad_points(P) * 6 * sizeof(double), capturing));
    for (int b = 0; b < G.tp.B; ++b)
      if (const int rc = track_object_lw<decltype(h)::value, BA>(tw, L, G, b, st, err)) return rc;
    return 0;
  });
}

// ---------------------------------------------------------------------------------------------------------------------
// Joint map-and-pose step (vmb_joint_step_lw): the layer-wise MAPPING step fed from camera-frame samples, with K11's
// per-ray rows taken from that step's own backward.  Per object b, in order on `st`:
//   k_joint_world  p = pose_point(T_f, q, 1) per point, f = the frame of the ray's draw (ba_draw_frame); k_lw_pe's
//                  t = p / scale is then bit-identical to the t that k_tlw_pose recomputes.  A ray whose frame is outside
//                  its table keeps p = q (identity pose), gets zero rows and sets VMB_BA_ST_BAD_FRAME.  Writes ctl (row
//                  ok = 1, scale[b]) for the pose kernels.
//   step_object    the training step on p, unchanged (forward, render, loss, weight-gradient GEMMs, dE); no AdamW here,
//                  because the pose terms read the PE directions from the fp32 param row and must see them before the update.
//   k_tlw_pose / k_tlw_reduce (BA flavour) on the training workspace's dE: one row per ray, loss columns 0.
// ---------------------------------------------------------------------------------------------------------------------
struct JointWorkspace {        // handle scratch (DeviceBuffer's rule); each step grows the buffers it uses
  DeviceBuffer<float> pw;      // [P][3] world points of the current object (fused step: of all B objects)
  DeviceBuffer<int> ctl;       // [8] as TrackWorkspace::ctl (only row ok and scale are read; layer-wise step)
  DeviceBuffer<double> gpt;    // [P][6] per-point pose terms (layer-wise step)
  DeviceBuffer<float> jdt;     // [P][2][3] the fused step's per-point dL/dt halves
};

// object o.b + blockIdx.y of a batched launch (the fused joint step: all B objects in one grid; the layer-wise step
// launches one object with gridDim.y = 1): its slice of the samples and of the draw tables
__device__ __forceinline__ TlwObj joint_obj(TlwObj o, long long pcs_stride, long long kf_draw_stride) {
  const int y = blockIdx.y;
  o.b += y; o.pcs += y * pcs_stride; o.kf_draw += y * kf_draw_stride; o.kf_frame += (size_t)y * o.kf_stride;
  return o;
}

// pw / pw_out: [gridDim.y][P][3]; ctl (layer-wise step only) gets row ok = 1 and scale[o.b]
__global__ void __launch_bounds__(256) k_joint_world(TlwObj o0, long long pcs_stride, long long kf_draw_stride,
                                                     const float* __restrict__ scale, float* __restrict__ pw,
                                                     float* __restrict__ pw_out, int* __restrict__ ctl) {
  ptx::pdl_wait();
  ptx::pdl_launch_dependents();
  const TlwObj o = joint_obj(o0, pcs_stride, kf_draw_stride);
  const long long P = (long long)o.R * o.S;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p == 0 && ctl) { ctl[3] = 1; ctl[4] = __float_as_int(scale[o.b]); }
  if (p >= P) return;
  pw += (size_t)blockIdx.y * P * 3;
  if (pw_out) pw_out += (size_t)blockIdx.y * P * 3;
  const int f = tlw_frame<true>(o, (int)(p / o.S));
  const float3 q = make_float3(o.pcs[p * 3], o.pcs[p * 3 + 1], o.pcs[p * 3 + 2]);
  const float3 w = f >= 0 ? pose_point(o.pose + (size_t)f * 16, q, 1.0f) : q;
  if (f < 0 && p % o.S == 0 && o.status) atomicOr(o.status, VMB_BA_ST_BAD_FRAME);
  pw[p * 3] = w.x; pw[p * 3 + 1] = w.y; pw[p * 3 + 2] = w.z;
  if (pw_out) { pw_out[p * 3] = w.x; pw_out[p * 3 + 1] = w.y; pw_out[p * 3 + 2] = w.z; }
}

// The fused joint step's rows (vmb_joint_step_fused): one thread per ray of object blockIdx.y, its samples in order,
// dL/dt = the two halves of jdt [B][R * S][2][3] added (hsel 0 + hsel 1), then pose_terms from the fp64 pose of the
// draw's frame; K11's row layout with the loss columns and column 9 at 0.  A ray whose frame is outside its table gets a
// zero row and sets VMB_BA_ST_BAD_FRAME.
__global__ void __launch_bounds__(128) k_joint_rows(TlwObj o0, long long pcs_stride, long long kf_draw_stride,
                                                    const float* __restrict__ scale, const float* __restrict__ jdt,
                                                    double* __restrict__ rows) {
  const TlwObj o = joint_obj(o0, pcs_stride, kf_draw_stride);
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= o.R) return;
  const int f = tlw_frame<true>(o, r);
  double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (f >= 0) {
    const double* T = o.pose + (size_t)f * 16;
    const float sc = scale[o.b];
    const float* h = jdt + ((size_t)blockIdx.y * o.R + r) * o.S * 6;
    for (int i = 0; i < o.S; ++i, h += 6) {
      const long long p = (long long)r * o.S + i;
      const float3 dt = make_float3(h[0] + h[3], h[1] + h[4], h[2] + h[5]);
      double c6[6];
      pose_terms(T, make_double3(o.pcs[p * 3], o.pcs[p * 3 + 1], o.pcs[p * 3 + 2]), dt, sc, c6);
#pragma unroll
      for (int c = 0; c < 6; ++c) s[c] += c6[c];
    }
  } else if (o.status) {
    atomicOr(o.status, VMB_BA_ST_BAD_FRAME);
  }
  double* dst = rows + ((size_t)blockIdx.y * o.R + r) * VMB_TRACK_PART;
#pragma unroll
  for (int c = 0; c < 6; ++c) dst[c] = s[c];
#pragma unroll
  for (int c = 6; c < VMB_TRACK_PART; ++c) dst[c] = 0.0;
}

// sp: the mapping step's arguments (pcs = camera-frame points); x: the per-draw pose tables and the output rows
template <int H>
static int joint_object_lw(Workspace& ws, JointWorkspace& jw, const VmbLayout& L, const StepParams& sp, const BaRays& x,
                           const double* poses, int* status, const __half* image, int b, float* pw_out, cudaStream_t st,
                           std::string& err) {
  const long long np = (long long)sp.R * sp.S;
  TlwObj o;
  memset(&o, 0, sizeof(o));
  o.b = b; o.R = sp.R; o.S = sp.S; o.n_rows = sp.B; o.pcs = sp.pcs + (size_t)b * sp.pcs_stride; o.pose = poses; o.status = status;
  o.n_pix_draw = x.n_pix_draw; o.n_poses = x.n_poses; o.kf_stride = x.kf_stride;
  o.kf_draw = x.kf_draw + (size_t)b * x.kf_draw_stride;
  o.kf_frame = x.kf_frame + (size_t)b * x.kf_stride;
  LW_TRY(launch_k(k_joint_world, dim3((unsigned)((np + 255) / 256)), dim3(256), 0, st, o, 0LL, 0LL, sp.scale, jw.pw,
                  pw_out ? pw_out + (size_t)b * np * 3 : nullptr, jw.ctl));
  StepParams s1 = sp;
  s1.pcs = jw.pw; s1.pcs_stride = 0;                // step_object reads object b's points at pcs + b * pcs_stride
  const int rc = step_object<H>(ws, L, s1, image, b, st, err);
  if (rc) return rc;
  int dev = 0;
  cudaGetDevice(&dev);
  LW_TRY(smem_limit_once<k_tlw_pose<true>>(dev, PEB_SMEM));
  // after step_object's join with its side stream: an ordinary launch
  LW_TRY(launch_k(k_tlw_pose<true>, dim3((unsigned)((np + 127) / 128)), dim3(128), (size_t)PEB_SMEM, st, o,
                  sp.params + (size_t)b * L.stride, (const int*)jw.ctl, L.o_B, (const float*)ws.dE, jw.gpt));
  if (pdl_ok(np)) pdl_arm();
  LW_TRY(launch_k(k_tlw_reduce<true>, dim3((sp.R + 127) / 128), dim3(128), 0, st, o, 1, sp.R, (const int*)jw.ctl,
                  (const double*)jw.gpt, (const double*)nullptr, x.rows + (size_t)b * sp.R * VMB_TRACK_PART));
  LW_TRY(cudaGetLastError());
  return 0;
}

static int launch_joint_lw(Workspace& ws, JointWorkspace& jw, const VmbLayout& L, const StepParams& sp, const BaRays& x,
                           const double* poses, int* status, const void* image, float* pw_out, cudaStream_t st,
                           std::string& err) {
  return for_hidden(L.H, "joint step", err, [&](auto h) -> int {
    const long long np = (long long)sp.R * sp.S, Pp = pad_points(np);
    const bool capturing = stream_capturing(st);
    LW_TRY(ws.grow(np, L.H, capturing));
    LW_TRY(jw.pw.grow((size_t)Pp * 3 * sizeof(float), capturing));
    LW_TRY(jw.ctl.grow(8 * sizeof(int), capturing));
    LW_TRY(jw.gpt.grow((size_t)Pp * 6 * sizeof(double), capturing));
    for (int b = 0; b < sp.B; ++b)
      if (const int rc = joint_object_lw<decltype(h)::value>(ws, jw, L, sp, x, poses, status, (const __half*)image, b, pw_out,
                                                             st, err))
        return rc;
    return 0;
  });
}
#undef LW_TRY

}  // namespace lw
