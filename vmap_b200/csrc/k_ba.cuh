// K11: bundle adjustment of keyframe poses against the object map -- pose-only passes against a frozen map, run between
// mapping frames.  The step is K10's (k_track.cuh) with a pose per ray; the update is one Adam / Exp over every frame
// of the pass's window.  The parts of the rule K10 shares (frame lookup, point, per-ray loss, pose terms, Adam / Exp)
// are the helpers of k_track.cuh.
//
// The rule (oracle/ba_oracle.py restates it):
//   Samples  each object of the mapping stack samples its own keyframe table with K3 in the mapping layout,
//            n_iter * win_size draws of n_samples_per_frame pixels (the do_bg background: n_iter * win_size_bg draws
//            of n_samples_per_frame_bg pixels from its own keyframe copies), in the camera frame (the keyframe's pose
//            taken as identity, so pcs holds q = d_c * z as K10's samples do), recording the keyframe index of each
//            draw.  Iteration i uses rays [i * n_per_optim, (i + 1) * n_per_optim) of each object (train.py:271).
//   Pose     a ray's pose is T_wc[f], f = kf_frame[object][keyframe index of its draw], a row of the fp64 pose table;
//            p = R_f q + t_f in fp32 from an fp32 copy of the pose, as K10.
//   Loss     K10's, unchanged: per object sum_b (L_d + 5 L_c + 10 L_o) over its iteration slice, var detached, each
//            ray's render and loss in fp64, the empty-mask rule per object and per term; summed over every object.
//   Gradient left perturbation per frame: dL/drho_f = sum g, dL/dphi_f = sum (R_f q) x g over the rays whose draw used
//            frame f, across every object and group.  Per-point terms fp32, the cross product fp64.  The step writes
//            one fp64 row per ray (its samples in order); the update sums each (object, draw) segment's rays in order,
//            then each frame's segments in (group, object, draw) order.  No floating-point atomics: results are
//            bitwise reproducible, eager or replayed.
//   Update   one Adam over the stacked tangents of the window frames, no weight decay, moments reset at iteration 1
//            of each pass, bias correction by the pass's iteration; a window frame no ray saw has gradient 0 (its
//            momentum still moves it).  R_f <- Exp(dphi) R_f, t_f <- t_f + drho in fp64 (pose_adam_exp).  `hold` (frame
//            0, the caller's anchor) never moves.  A non-finite loss, window gradient or window pose skips the whole
//            iteration's update (at iteration 1 the moments are still reset) and sets VMB_ST_NONFINITE.
//   Write-back after the last iteration, each window frame's pose goes in fp32 to every entry i of each target
//            (the frame store's slots, the background's keyframe copies) whose frame_of[i] is that frame.
//   Guards   a draw whose keyframe index or frame id is outside its table contributes nothing and sets
//            VMB_BA_ST_BAD_FRAME (so does a window entry >= n_poses); a row outside the stack sets
//            VMB_TRACK_ST_BAD_ROW, as K10.
#pragma once
#include "k_track.cuh"

template <int H, int TP>
__global__ void __launch_bounds__(128, 1) k_ba_step(TrackParams a, VmbLayout L, BaRays x) {
  track_step_body<H, TP, true>(a, L, x);
}

struct BaGroupDev {
  const double* rows;            // [n_obj][n_rays][VMB_TRACK_PART]
  int n_obj, n_rays, n_pix_draw;
  const int* kf_draw; long long kf_draw_stride;
  const int* kf_frame; int kf_stride;
};

struct BaTargetDev { const int* frame_of; float* t_wc; int n; };

struct BaUpdateParams {
  int n_groups;
  BaGroupDev g[VMB_TRACK_MAX_GROUPS];
  int iter, n_iter;              // 1-based iteration of this pass
  int n_poses, n_win, hold;
  const int* win;                // [n_win] frame ids, -1 = padding
  double* pose;                  // [n_poses][16] in/out
  double* adam;                  // [n_win][12]
  double* scratch;               // [segments][8] | [n_win][6]
  PoseUpdateScalars s;
  double* loss;                  // optional [n_iter]
  double* pose_hist;             // optional [n_iter+1][n_win][16]
  double* grad_hist;             // optional [n_iter][n_win][6]
  BaTargetDev tgt[2];
  int* status;
};

__global__ void __launch_bounds__(256) k_ba_update(BaUpdateParams a) {
  constexpr int NT = 256;
  __shared__ int s_bad;
  __shared__ double s_loss;
  const int tid = threadIdx.x;
  if (tid == 0) s_bad = 0;
  int n_seg = 0;
  for (int gi = 0; gi < a.n_groups; ++gi) n_seg += a.g[gi].n_obj * (a.g[gi].n_rays / a.g[gi].n_pix_draw);
  double* seg = a.scratch;                        // grad[6], weighted loss, frame id (-1: contributes to no frame)
  double* gw = a.scratch + (size_t)n_seg * 8;

  // ---- one segment = the n_pix_draw rays of one draw of one object, summed in ray order ----------------------------
  for (int s = tid; s < n_seg; s += NT) {
    int gi = 0, base = 0;
    while (s >= base + a.g[gi].n_obj * (a.g[gi].n_rays / a.g[gi].n_pix_draw)) {
      base += a.g[gi].n_obj * (a.g[gi].n_rays / a.g[gi].n_pix_draw);
      ++gi;
    }
    const BaGroupDev& G = a.g[gi];
    const int nd = G.n_rays / G.n_pix_draw, ob = (s - base) / nd, d = (s - base) - ob * nd;
    const double* r = G.rows + ((size_t)ob * G.n_rays + (size_t)d * G.n_pix_draw) * VMB_TRACK_PART;
    double acc[9];
#pragma unroll
    for (int c = 0; c < 9; ++c) acc[c] = 0.0;
    for (int i = 0; i < G.n_pix_draw; ++i)
#pragma unroll
      for (int c = 0; c < 9; ++c) acc[c] += r[(size_t)i * VMB_TRACK_PART + c];
    const int f = ba_draw_frame(G.kf_draw, G.kf_draw_stride, G.kf_frame, G.kf_stride, a.n_poses, ob, d);
    double* o = seg + (size_t)s * 8;
    for (int c = 0; c < 6; ++c) o[c] = acc[c];
    o[6] = acc[6] + a.s.cs * acc[7] + a.s.os * acc[8];
    o[7] = (double)f;
  }
  __syncthreads();
  if (tid == 0) {
    double L = 0.0;
    for (int s = 0; s < n_seg; ++s) L += seg[(size_t)s * 8 + 6];
    s_loss = L;
    if (a.loss) a.loss[a.iter - 1] = L;
  }

  // ---- per window frame: its segments in (group, object, draw) order -----------------------------------------------
  for (int w = tid; w < a.n_win; w += NT) {
    const int f = a.win[w];
    const bool live = f >= 0 && f < a.n_poses && f != a.hold;
    if (f >= a.n_poses && a.status) atomicOr(a.status, VMB_BA_ST_BAD_FRAME);
    double g[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    bool ok = true;
    if (live) {
      const double fd = (double)f;
      for (int s = 0; s < n_seg; ++s) {
        const double* o = seg + (size_t)s * 8;
        if (o[7] == fd)
#pragma unroll
          for (int c = 0; c < 6; ++c) g[c] += o[c];
      }
      const double* T = a.pose + (size_t)f * 16;
      for (int c = 0; c < 6; ++c) ok = ok && isfinite(g[c]);
      for (int i = 0; i < 16; ++i) ok = ok && isfinite(T[i]);
      if (a.pose_hist && a.iter == 1)
        for (int i = 0; i < 16; ++i) a.pose_hist[(size_t)w * 16 + i] = T[i];
    }
    for (int c = 0; c < 6; ++c) gw[(size_t)w * 6 + c] = g[c];
    if (a.grad_hist)
      for (int c = 0; c < 6; ++c) a.grad_hist[((size_t)(a.iter - 1) * a.n_win + w) * 6 + c] = g[c];
    if (!ok) atomicOr(&s_bad, 1);
  }
  __syncthreads();
  const bool ok = !s_bad && isfinite(s_loss);
  if (!ok && tid == 0 && a.status) atomicOr(a.status, VMB_ST_NONFINITE);

  // ---- Adam + Exp per window frame (each thread owns the same entries as above) ------------------------------------
  for (int w = tid; w < a.n_win; w += NT) {
    const int f = a.win[w];
    const bool live = f >= 0 && f < a.n_poses && f != a.hold;
    double* A = a.adam + (size_t)w * 12;
    if (live && ok) {
      double* P = a.pose + (size_t)f * 16;
      double T[16];
      for (int i = 0; i < 16; ++i) T[i] = P[i];
      pose_adam_exp(T, A, gw + (size_t)w * 6, a.iter, a.s);
      for (int i = 0; i < 16; ++i) P[i] = T[i];
    } else {
      pose_adam_skip(A, a.iter);
    }
    if (!live) continue;
    const double* P = a.pose + (size_t)f * 16;
    if (a.pose_hist)
      for (int i = 0; i < 16; ++i) a.pose_hist[((size_t)a.iter * a.n_win + w) * 16 + i] = P[i];
    if (a.iter == a.n_iter)
      for (int t = 0; t < 2; ++t) {
        const BaTargetDev& D = a.tgt[t];
        if (!D.t_wc) continue;
        for (int i = 0; i < D.n; ++i)
          if (D.frame_of[i] == f)
            for (int k = 0; k < 16; ++k) D.t_wc[(size_t)i * 16 + k] = (float)P[k];
      }
  }
}
