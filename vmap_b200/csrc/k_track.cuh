// K10: camera tracking against the object map -- pose gradient through every tracked object's network and an
// on-device Adam / Exp pose optimiser.  CUDA-core fp32 for the networks: K1 fp32's network (NetTile of k_step_fp32.cuh:
// tile, embedding, forward and input gradients), no weight gradients; fp64 for the pose, the partial sums and the update.
//
// The rule (oracle/track_oracle.py restates it).  The parts K11 (k_ba.cuh) and the layer-wise path (k_track_lw.cuh)
// share are written once below, as the helpers ba_draw_frame, pose_point, ray_loss, pose_terms and pose_adam_exp, with
// the mask counts of k_step_fp32.cuh (slice_mask_count); each kernel keeps only its own reductions.
//   Pose     camera-to-world T_wc = [R | t] (the reference's twc), fp64 [4][4] row-major in device memory.
//   Samples  each tracked object samples the frame once in the camera frame (K3's camera_frame mode: the points of an
//            IDENTITY pose; one keyframe: the new frame's slot and the object's 2-D box from this frame's ingest; the
//            background, id 0, uses the full frame; n_bins_cam2surface 1 for objects, 5 for the background), so pcs holds camera-frame points
//            q = d_c * z, with z, gt_depth, gt_colour, sem and mask_depth in the training rule (vmap.py:366-459).
//            n_iter draws of n_pix rays; iteration i uses draw i (train.py:271).
//   Points   p = R q + t - obj_center (obj_center = 0 in the package), in fp32 from an fp32 copy of the pose; the
//            network sees p / scale (embedding.py:80).
//   Loss     the training loss of every tracked object, sum_b (L_d + 5 L_c + 10 L_o) (loss.py:5-62,
//            render_rays.py:53-96), var detached (loss.py:29), with each ray's render and loss in fp64.  Empty masks
//            are handled PER OBJECT AND PER TERM: a term whose own mask count is 0 contributes 0 for that object only
//            (the reference zeroes the term for the whole batch, render_rays.py:68-73, which would stop tracking whenever one small object has no valid ray).
//   Gradient left perturbation R <- Exp(phi) R, t <- t + rho:
//              dL/drho = sum g,  dL/dphi = sum (R q) x g,  g = dL/dp
//              g = (1/scale) (dL/de_xyz + sum_{k,d} dL/de_{k,d} * pi 2^k cos(pi 2^k proj_d) * B_d)
//            per-point terms in fp32, (R q) x g in fp64 from the fp64 pose; per-CTA partials summed in fp64 in point
//            order, no floating-point atomics; the update sums every group's partials in (group, object, tile) order
//            through a fixed tree.  Results are bitwise reproducible.
//   Update   Adam on the tangent (phi, rho), no weight decay: m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2 (m = v = 0
//            before iteration 1 of each frame), m^ = m / (1 - b1^i), v^ = v / (1 - b2^i),
//            delta = -lr * m^ / (sqrt(v^) + eps) with lr = (lr_rot x 3, lr_trans x 3);
//            R <- Exp(delta_phi) R, t <- t + delta_rho.  Exp = Rodrigues in fp64, I + [phi]x below |phi| = 1e-12.
//            A non-finite loss, gradient or pose skips the iteration's update (moments included; at iteration 1 the
//            moments are still reset to 0) and sets VMB_ST_NONFINITE.
#pragma once
#include "common.cuh"
#include "k_step_fp32.cuh"

// VMB_TRACK_PART (doubles per CTA partial row: dL/dphi[3], dL/drho[3], L_d, L_c, L_o, 0), VMB_TRACK_MAX_GROUPS and
// VMB_TRACK_ST_BAD_ROW (a rows[] entry outside [0, n_rows); that object contributes nothing) are in vmap_b200.h.

struct TrackParams {
  int B, R, S, n_rows;
  const int* rows;
  const float* pcs;  long long pcs_stride;
  const float* z;    long long z_stride;
  const float* gt_depth;  long long gt_depth_stride;
  const float* gt_colour; long long gt_colour_stride;
  const unsigned char* sem;  long long sem_stride;
  const unsigned char* mask; long long mask_stride;
  const float* params;
  const float* scale;
  const double* pose;
  double* partials;              // [B][tiles][VMB_TRACK_PART]
  float cs, os;
  int* status;
};

// rows [j0, j0 + OB) of d(loss)/d(embedding) for one point: acc[jj] = sum_o dy[o] W[o*ld + jj] (+ the second operand)
// folded into d(loss)/d(t), t = p / scale.  Rows past `jend` are computed (they read inside the param row) and dropped.
template <int OB>
__device__ __forceinline__ void pe_input_grad(const float (&acc)[OB], int j0, int jend, const float* __restrict__ Bm,
                                              float t0, float t1, float t2, float (&dt)[3]) {
#pragma unroll
  for (int jj = 0; jj < OB; ++jj) {
    const int j = j0 + jj;
    if (j >= jend) break;
    if (j < 3) {                                              // xyz rows (constant indices keep dt in registers)
      dt[0] += (j == 0) ? acc[jj] : 0.f; dt[1] += (j == 1) ? acc[jj] : 0.f; dt[2] += (j == 2) ? acc[jj] : 0.f;
      continue;
    }
    const int k = (j - 3) / VMB_NDIRS, d = (j - 3) - k * VMB_NDIRS;
    const float* Bd = Bm + d * 3;
    const float b0 = __ldg(Bd), b1 = __ldg(Bd + 1), b2 = __ldg(Bd + 2);
    const float proj = fmaf(b2, t2, fmaf(b1, t1, b0 * t0));          // embedding.py:88
    const float fk = (float)(1 << k);
    const float arg = (proj * fk) * VMB_PI_F;
    const float c = (acc[jj] * cosf(arg) * VMB_PI_F) * fk;
    dt[0] = fmaf(c, b0, dt[0]); dt[1] = fmaf(c, b1, dt[1]); dt[2] = fmaf(c, b2, dt[2]);
  }
}

// K11's per-ray pose (k_ba.cuh): draw d of object b used keyframe index kf_draw[b][d], whose frame id (the row of the
// fp64 pose table a.pose) is kf_frame[b][kf].  K10 does not read it.
struct BaRays {
  const int* kf_draw; long long kf_draw_stride;     // [B][draws of the slice]
  const int* kf_frame; int kf_stride;               // [B][kf_stride], -1 = no frame
  int n_pix_draw, n_poses;                          // rays per draw, rows of the pose table
  double* rows;                                     // out [B][R][VMB_TRACK_PART] per-ray rows
};

// ---- the pose rule, written once for K10, K11 (k_ba.cuh) and the layer-wise path (k_track_lw.cuh) -----------------

// frame id of draw `d` of object `b`, or -1 when the keyframe index or the frame id is outside its table
__device__ __forceinline__ int ba_draw_frame(const int* kf_draw, long long kf_draw_stride, const int* kf_frame,
                                             int kf_stride, int n_poses, int b, int d) {
  const int kf = kf_draw[(size_t)b * kf_draw_stride + d];
  if (kf < 0 || kf >= kf_stride) return -1;
  const int f = kf_frame[(size_t)b * kf_stride + kf];
  return (f >= 0 && f < n_poses) ? f : -1;
}

// the network input of camera-frame point q: p = R q + t in fp32 from an fp32 copy of the fp64 pose T, then p / scale
__device__ __forceinline__ float3 pose_point(const double* T, float3 q, float sc) {
  const float x = fmaf((float)T[2], q.z, fmaf((float)T[1], q.y, (float)T[0] * q.x)) + (float)T[3];
  const float y = fmaf((float)T[6], q.z, fmaf((float)T[5], q.y, (float)T[4] * q.x)) + (float)T[7];
  const float w = fmaf((float)T[10], q.z, fmaf((float)T[9], q.y, (float)T[8] * q.x)) + (float)T[11];
  return make_float3(x / sc, y / sc, w / sc);
}

// one point's pose terms c = ((R q) x g, g) in fp64 from the fp64 pose, g = dL/dt / scale (q: the fp32 point, widened)
__device__ __forceinline__ void pose_terms(const double* T, double3 q, float3 dt, float sc, double (&c)[6]) {
  const double g0 = (double)(dt.x / sc), g1 = (double)(dt.y / sc), g2 = (double)(dt.z / sc);
  const double x0 = T[0] * q.x + T[1] * q.y + T[2] * q.z;     // R q in fp64
  const double x1 = T[4] * q.x + T[5] * q.y + T[6] * q.z;
  const double x2 = T[8] * q.x + T[9] * q.y + T[10] * q.z;
  c[0] = x1 * g2 - x2 * g1; c[1] = x2 * g0 - x0 * g2; c[2] = x0 * g1 - x1 * g0;
  c[3] = g0; c[4] = g1; c[5] = g2;
}

// One ray's loss from its fp64 render (depth D, opacity O, colour C, detached variance V): the three loss terms
// L_d, L_c, L_o in fp64 and the fp32 upstream gradients d(loss)/d(D, C, O).  Empty masks are handled per object and per
// term: cnt[] are the object's slice counts (nd, no, ns), and a term whose count is 0 contributes 0.  A ray without a
// pose (rok false) is masked out of every term.
struct RayLoss { double l[3]; float gD, gC0, gC1, gC2, gO; };

__device__ __forceinline__ RayLoss ray_loss(double D, double O, double C0, double C1, double C2, double V, int sv,
                                            bool md, float gt_d, const float* gc, bool rok, const int (&cnt)[3],
                                            float cs, float os) {
  RayLoss r;
  const double m_o = (sv != 0 && rok) ? 1.0 : 0.0;
  const double m_s = (sv != 2 && rok) ? 1.0 : 0.0;
  const double m_d = md ? m_o : 0.0;
  const double gd = gt_d;
  const double inv_nd = cnt[0] ? 1.0 / ((double)cnt[0] + 1e-10) : 0.0;
  const double inv_no = cnt[1] ? 1.0 / ((double)cnt[1] + 1e-10) : 0.0;
  const double inv_ns = cnt[2] ? 1.0 / ((double)cnt[2] + 1e-10) : 0.0;
  const double info = 1.0 / (sqrt(V) + 1e-4);               // render_rays.py:74-79
  const double e_d = D - gd, e_o = O - m_o;
  const double e_c0 = C0 - (double)gc[0], e_c1 = C1 - (double)gc[1], e_c2 = C2 - (double)gc[2];
  r.l[0] = cnt[0] ? fabs(e_d) * m_d * info * inv_nd : 0.0;
  r.l[1] = cnt[1] ? (fabs(e_c0) + fabs(e_c1) + fabs(e_c2)) * m_o * inv_no : 0.0;
  r.l[2] = cnt[2] ? fabs(e_o) * m_s * inv_ns : 0.0;
  r.gD = (float)(m_d * info * inv_nd) * vmb_sign((float)e_d);
  const float kc = (float)((double)cs * m_o * inv_no);
  r.gC0 = kc * vmb_sign((float)e_c0); r.gC1 = kc * vmb_sign((float)e_c1); r.gC2 = kc * vmb_sign((float)e_c2);
  r.gO = (float)((double)os * m_s * inv_ns) * vmb_sign((float)e_o);
  return r;
}

// One CTA = one tile of whole rays of one tracked object (blockIdx.y): NetTile's tile, embedding, forward and input
// gradients (k_step_fp32.cuh), so the pose gradient is that of the network K1 fp32 trains.
// BA = false is K10 (one pose, per-CTA partials); BA = true is K11 (a pose per ray, per-ray rows).
template <int H, int TP, bool BA>
__device__ __forceinline__ void track_step_body(const TrackParams& a, const VmbLayout& L, const BaRays& x) {
  using Net = NetTile<H, TP>;
  constexpr int NT = Net::NT, PT = Net::PT, NOG = Net::NOG, OB = Net::OB;
  extern __shared__ float sm[];
  const Net net(sm, L, a.S, a.R);         // net.sHd's 12 rows are followed by the dt partials
  __shared__ double s_g[6][TP];           // per-point pose-gradient terms
  __shared__ double s_l[3][TP];           // per-ray loss terms
  __shared__ int s_cnt[3][NT / 32];

  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int S = a.S, R = a.R;
  double* part = a.partials + ((size_t)b * gridDim.x + blockIdx.x) * VMB_TRACK_PART;
  const int row = a.rows[b];
  if (row < 0 || row >= a.n_rows) {                   // uniform over the CTA
    if constexpr (BA) {
      if (tid < net.nr && net.r0 + tid < R)
        for (int c = 0; c < VMB_TRACK_PART; ++c) x.rows[((size_t)b * R + net.r0 + tid) * VMB_TRACK_PART + c] = 0.0;
    } else if (tid < VMB_TRACK_PART) {
      part[tid] = 0.0;
    }
    if (tid == 0 && a.status) atomicOr(a.status, VMB_TRACK_ST_BAD_ROW);
    return;
  }
  const float* __restrict__ P = a.params + (size_t)row * L.stride;

  // ---- per-object mask counts of this slice (loss.py:16-18,38): every CTA of the object counts the same rays --------
  {
    const unsigned char* sv = a.sem + (size_t)b * a.sem_stride;
    const unsigned char* mv = a.mask + (size_t)b * a.mask_stride;
    int nd = 0, no = 0, ns = 0;
    for (int r = tid; r < R; r += NT) slice_mask_count(sv, mv, r, nd, no, ns);
    warp_mask_counts(tid, nd, no, ns, s_cnt);
  }

  // ---- A: point p = R q + t (fp32 copy of the fp64 pose), positional embedding of p / scale ---------------------------
  const double* T = a.pose;
  bool pok = net.pvalid;                              // K11: the ray's frame is in the pose table
  if constexpr (BA) {
    const int f = net.pvalid ? ba_draw_frame(x.kf_draw, x.kf_draw_stride, x.kf_frame, x.kf_stride, x.n_poses, b,
                                             (net.r0 + net.rl) / x.n_pix_draw) : -1;
    pok = f >= 0;
    T = a.pose + (size_t)(pok ? f : 0) * 16;
  }
  float3 q = make_float3(0.f, 0.f, 0.f), t = q;
  const float sc = a.scale[row];
  if (pok) {
    const size_t gi = (size_t)b * a.pcs_stride + ((size_t)(net.r0 + net.rl) * S + net.sidx) * 3;
    q = make_float3(a.pcs[gi], a.pcs[gi + 1], a.pcs[gi + 2]);
    t = pose_point(T, q, sc);
  }
  if (net.og == 0) {
    net.sE[0 * PT + net.p] = t.x; net.sE[1 * PT + net.p] = t.y; net.sE[2 * PT + net.p] = t.z;
    net.sHd[8 * PT + net.p] = net.pvalid ? a.z[(size_t)b * a.z_stride + (size_t)(net.r0 + net.rl) * S + net.sidx] : 0.f;
    net.sHd[4 * PT + net.p] = 0.f; net.sHd[5 * PT + net.p] = 0.f; net.sHd[6 * PT + net.p] = 0.f; net.sHd[7 * PT + net.p] = 0.f;
  }
  net.embed(P, L, t);

  // ---- B: MLP forward (model.py:54-85) -------------------------------------------------------------------------------
  net.forward(P, L);

  // ---- C: render + loss + d(loss)/d(alpha, colour), per-object per-term empty-mask rule ------------------------------
  if (tid < TP) { s_l[0][tid] = 0.0; s_l[1][tid] = 0.0; s_l[2][tid] = 0.0; }
  if (tid < net.nr && net.r0 + tid < R) {    // per-ray sums in fp64: depth and variance cancel when a ray's weight
    const int ray = net.r0 + tid;             // sits on one sample, and the depth weight 1/(sqrt(var)+1e-4) amplifies it
    const int pb = tid * S;
    double Tr = 1.0, D = 0.0, O = 0.0, C0 = 0.0, C1 = 0.0, C2 = 0.0;
    for (int s = 0; s < S; ++s) {
      const int qi = pb + s;
      const float occ = vmb_sigmoid(net.sHd[0 * PT + qi]);  // render_rays.py:6
      const double w = (double)occ * Tr;                    // render_rays.py:34
      net.sHd[9 * PT + qi] = occ; net.sHd[10 * PT + qi] = (float)Tr; net.sHd[11 * PT + qi] = (float)w;
      D += w * (double)net.sHd[8 * PT + qi]; O += w;
      C0 += w * (double)net.sHd[1 * PT + qi]; C1 += w * (double)net.sHd[2 * PT + qi]; C2 += w * (double)net.sHd[3 * PT + qi];
      Tr *= ((double)vmb_sigmoid(-net.sHd[0 * PT + qi]) + 1e-10);  // render_rays.py:29, 1 - occ as sigmoid(-alpha):
    }                                                       // no cancellation where occ rounds to 1 in fp32
    double V = 0.0;
    for (int s = 0; s < S; ++s) {
      const double dz = (double)net.sHd[8 * PT + pb + s] - D;
      V += (double)net.sHd[11 * PT + pb + s] * dz * dz;     // loss.py:28-29 (detached)
    }
    int cnt[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) cnt[c] = s_cnt[c][0] + s_cnt[c][1] + s_cnt[c][2] + s_cnt[c][3];
    const int sv = a.sem[(size_t)b * a.sem_stride + ray];
    bool rok = true;                          // K11: a ray whose frame is outside the pose table contributes nothing
    if constexpr (BA) {
      rok = ba_draw_frame(x.kf_draw, x.kf_draw_stride, x.kf_frame, x.kf_stride, x.n_poses, b, ray / x.n_pix_draw) >= 0;
      if (!rok && a.status) atomicOr(a.status, VMB_BA_ST_BAD_FRAME);
    }
    const RayLoss ls = ray_loss(D, O, C0, C1, C2, V, sv,
                                a.mask[(size_t)b * a.mask_stride + ray] != 0, a.gt_depth[(size_t)b * a.gt_depth_stride + ray],
                                a.gt_colour + (size_t)b * a.gt_colour_stride + (size_t)ray * 3, rok, cnt, a.cs, a.os);
    s_l[0][tid] = ls.l[0]; s_l[1][tid] = ls.l[1]; s_l[2][tid] = ls.l[2];
    const float gD = ls.gD, gC0 = ls.gC0, gC1 = ls.gC1, gC2 = ls.gC2, gO = ls.gO;
    float suffix = 0.f;
    for (int s = S - 1; s >= 0; --s) {
      const int qi = pb + s;
      const float occ = net.sHd[9 * PT + qi], Ts = net.sHd[10 * PT + qi], w = net.sHd[11 * PT + qi];
      const float c0 = net.sHd[1 * PT + qi], c1 = net.sHd[2 * PT + qi], c2 = net.sHd[3 * PT + qi];
      const float Gs = fmaf(gD, net.sHd[8 * PT + qi], fmaf(gC0, c0, fmaf(gC1, c1, fmaf(gC2, c2, gO))));
      const float fr = vmb_sigmoid(-net.sHd[0 * PT + qi]); // 1 - occ
      const float f = fr + 1e-10f;
      const float docc = Gs * Ts - suffix / f;
      net.sHd[4 * PT + qi] = 10.0f * docc * occ * fr;
      net.sHd[5 * PT + qi] = gC0 * w * c0 * (1.f - c0);
      net.sHd[6 * PT + qi] = gC1 * w * c1 * (1.f - c1);
      net.sHd[7 * PT + qi] = gC2 * w * c2 * (1.f - c2);
      suffix = fmaf(Gs, w, suffix);
    }
  }
  __syncthreads();

  // ---- D: backward to the inputs only (no weight gradients) ----------------------------------------------------------
  net.dyc(P, L);
  net.dy4(P, L);
  net.dgrad(net.sA3, net.sA4, P + L.o_Wm2, H);                                // dY3
  net.dgrad(net.sA2, net.sA3, P + L.o_Wcat, H + VMB_E1);                      // dY2
  net.dgrad(net.sA1, net.sA2, P + L.o_Wm1, H);                                // dY1

  // d(loss)/d(t): embedding rows in blocks of OB, rows [0, 87) through in_layer + cat_layer, [87, E) through color_linear
  {
    float dt[3] = {0.f, 0.f, 0.f};
    const int nb1 = (VMB_E1 + OB - 1) / OB, nb2 = (L.e2 + OB - 1) / OB;
    const int ldc = H + VMB_E1, ldl = H + L.e2;
    for (int blk = net.og; blk < nb1 + nb2; blk += NOG) {
      float acc[OB];
#pragma unroll
      for (int j = 0; j < OB; ++j) acc[j] = 0.f;
      if (blk < nb1) {
        const int j0 = blk * OB;
        dgrad_block<OB>(acc, P + L.o_Win + j0, VMB_E1, net.sA1 + net.p, H, PT);
        dgrad_block<OB>(acc, P + L.o_Wcat + H + j0, ldc, net.sA3 + net.p, H, PT);
        pe_input_grad<OB>(acc, j0, VMB_E1, P + L.o_B, t.x, t.y, t.z, dt);
      } else {
        const int j0 = (blk - nb1) * OB;
        dgrad_block<OB>(acc, P + L.o_Wcl + H + j0, ldl, net.sAC + net.p, H, PT);
        pe_input_grad<OB>(acc, VMB_E1 + j0, L.E, P + L.o_B, t.x, t.y, t.z, dt);
      }
    }
    net.sHd[(net.og * 3 + 0) * PT + net.p] = dt[0];
    net.sHd[(net.og * 3 + 1) * PT + net.p] = dt[1];
    net.sHd[(net.og * 3 + 2) * PT + net.p] = dt[2];
  }
  __syncthreads();
  if (net.og == 0) {
    float d0 = 0.f, d1 = 0.f, d2 = 0.f;
#pragma unroll
    for (int g = 0; g < NOG; ++g) {
      d0 += net.sHd[(g * 3) * PT + net.p]; d1 += net.sHd[(g * 3 + 1) * PT + net.p]; d2 += net.sHd[(g * 3 + 2) * PT + net.p];
    }
    double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (pok) pose_terms(T, make_double3(q.x, q.y, q.z), make_float3(d0, d1, d2), sc, c);
#pragma unroll
    for (int i = 0; i < 6; ++i) s_g[i][net.p] = c[i];
  }
  __syncthreads();
  if constexpr (BA) {                                       // per-ray rows: the ray's samples in order
    if (tid < net.nr && net.r0 + tid < R) {
      double* out = x.rows + ((size_t)b * R + net.r0 + tid) * VMB_TRACK_PART;
      for (int c = 0; c < 6; ++c) {
        double s = 0.0;
        for (int i = 0; i < S; ++i) s += s_g[c][tid * S + i];
        out[c] = s;
      }
      out[6] = s_l[0][tid]; out[7] = s_l[1][tid]; out[8] = s_l[2][tid]; out[9] = 0.0;
    }
  } else if (tid < 6) {
    double s = 0.0;
    for (int i = 0; i < net.np; ++i) s += s_g[tid][i];
    part[tid] = s;
  } else if (tid < 9) {
    double s = 0.0;
    for (int i = 0; i < net.nr; ++i) s += s_l[tid - 6][i];
    part[tid] = s;
  } else if (tid == 9) {
    part[9] = 0.0;
  }
}

template <int H, int TP>
__global__ void __launch_bounds__(128, 1) k_track_step(TrackParams a, VmbLayout L) {
  track_step_body<H, TP, false>(a, L, BaRays{});
}

// ---------------------------------------------------------------------------------------------------------------------
// Update: one CTA of 256 threads.  Thread k sums the objects k, k + 256, ... of the concatenated (group, object) list,
// each object's tiles in order; a fixed tree joins the threads; thread 0 runs Adam + Exp.
// ---------------------------------------------------------------------------------------------------------------------
struct TrackGroupDev { const double* partials; int n_obj, tiles; float* loss_terms; };

// Adam's rates, betas, eps and bias corrections 1 - b^iter for the iteration, and the loss weights
struct PoseUpdateScalars {
  double lr[6], b1, b2, eps, bc1, bc2;
  double cs, os;
};

struct TrackUpdateParams {
  int n_groups;
  TrackGroupDev g[VMB_TRACK_MAX_GROUPS];
  int iter;                      // 1-based iteration of this frame
  double* pose;                  // [16] in/out
  double* adam;                  // [12] m, v (not read at iter 1)
  PoseUpdateScalars s;
  double* loss;                  // optional [n_iter]: loss[iter-1]
  double* pose_hist;             // optional [n_iter+1][16]
  double* grad_hist;             // optional [n_iter][6]
  int* status;
};

// Exp of so(3) by Rodrigues in fp64, I + [w]x below |w| = 1e-12
__device__ inline void pose_exp(const double (&w)[3], double (&E)[9]) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  const double th = sqrt(th2);
  double A, Bc;
  if (th < 1e-12) { A = 1.0; Bc = 0.0; }
  else { A = sin(th) / th; Bc = (1.0 - cos(th)) / th2; }
  const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double k2 = 0.0;
      for (int m = 0; m < 3; ++m) k2 += K[i * 3 + m] * K[m * 3 + j];
      E[i * 3 + j] = (i == j ? 1.0 : 0.0) + A * K[i * 3 + j] + Bc * k2;
    }
}

// One Adam step on the tangent (phi, rho) with gradient g[6] and moments A = m[6], v[6] (not read at iteration 1), then
// the left update R <- Exp(delta_phi) R, t <- t + delta_rho of the pose T (row-major [4][4]).
__device__ __forceinline__ void pose_adam_exp(double (&T)[16], double* A, const double* g, int iter,
                                              const PoseUpdateScalars& s) {
  double d[6];
  for (int c = 0; c < 6; ++c) {
    const double m = (iter == 1 ? 0.0 : s.b1 * A[c]) + (1.0 - s.b1) * g[c];
    const double v = (iter == 1 ? 0.0 : s.b2 * A[6 + c]) + (1.0 - s.b2) * g[c] * g[c];
    A[c] = m; A[6 + c] = v;
    d[c] = -s.lr[c] * (m / s.bc1) / (sqrt(v / s.bc2) + s.eps);
  }
  const double w[3] = {d[0], d[1], d[2]};
  double E[9];
  pose_exp(w, E);
  double Rn[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      Rn[i * 3 + j] = E[i * 3 + 0] * T[0 * 4 + j] + E[i * 3 + 1] * T[1 * 4 + j] + E[i * 3 + 2] * T[2 * 4 + j];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[i * 4 + j] = Rn[i * 3 + j];
    T[i * 4 + 3] += d[3 + i];
  }
}

// a skipped update still restarts the moments when it is the first iteration
__device__ __forceinline__ void pose_adam_skip(double* A, int iter) {
  if (iter == 1) for (int c = 0; c < 12; ++c) A[c] = 0.0;
}

__global__ void __launch_bounds__(256) k_track_update(TrackUpdateParams a) {
  constexpr int NC = 7;                                     // grad[6], loss
  __shared__ double s_acc[NC][256];
  const int tid = threadIdx.x;
  double acc[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) acc[c] = 0.0;
  int base = 0;
  for (int gi = 0; gi < a.n_groups; ++gi) {
    const TrackGroupDev G = a.g[gi];
    for (int ob = ((tid - base) % 256 + 256) % 256; ob < G.n_obj; ob += 256) {
      const double* pr = G.partials + (size_t)ob * G.tiles * VMB_TRACK_PART;
      double s[9];
#pragma unroll
      for (int c = 0; c < 9; ++c) s[c] = 0.0;
      for (int t = 0; t < G.tiles; ++t)
#pragma unroll
        for (int c = 0; c < 9; ++c) s[c] += pr[(size_t)t * VMB_TRACK_PART + c];
      const double tot = s[6] + a.s.cs * s[7] + a.s.os * s[8];
      if (G.loss_terms) {
        float* lt = G.loss_terms + (size_t)ob * 4;
        lt[0] = (float)s[6]; lt[1] = (float)s[7]; lt[2] = (float)s[8]; lt[3] = (float)tot;
      }
#pragma unroll
      for (int c = 0; c < 6; ++c) acc[c] += s[c];
      acc[6] += tot;
    }
    base += G.n_obj;
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) s_acc[c][tid] = acc[c];
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (tid < st)
#pragma unroll
      for (int c = 0; c < NC; ++c) s_acc[c][tid] += s_acc[c][tid + st];
    __syncthreads();
  }
  if (tid != 0) return;

  double g[6];
  for (int c = 0; c < 6; ++c) g[c] = s_acc[c][0];
  const double loss = s_acc[6][0];
  if (a.loss) a.loss[a.iter - 1] = loss;
  if (a.grad_hist) for (int c = 0; c < 6; ++c) a.grad_hist[(size_t)(a.iter - 1) * 6 + c] = g[c];
  double T[16];
  for (int i = 0; i < 16; ++i) T[i] = a.pose[i];
  if (a.pose_hist && a.iter == 1) for (int i = 0; i < 16; ++i) a.pose_hist[i] = T[i];
  bool ok = isfinite(loss);
  for (int c = 0; c < 6; ++c) ok = ok && isfinite(g[c]);
  for (int i = 0; i < 16; ++i) ok = ok && isfinite(T[i]);
  if (ok) {
    pose_adam_exp(T, a.adam, g, a.iter, a.s);
    for (int i = 0; i < 16; ++i) a.pose[i] = T[i];
  } else {
    pose_adam_skip(a.adam, a.iter);
    if (a.status) atomicOr(a.status, VMB_ST_NONFINITE);
  }
  if (a.pose_hist) for (int i = 0; i < 16; ++i) a.pose_hist[(size_t)a.iter * 16 + i] = T[i];
}
