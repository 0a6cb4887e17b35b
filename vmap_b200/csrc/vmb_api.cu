// C ABI of libvmap_b200.so (see include/vmap_b200.h).  Host-side launch logic only.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/vmap_b200.h"
#include "common.cuh"
#include "k_step_fp32.cuh"
#include "k_adam.cuh"
#include "k_sampler.cuh"
#include "k_ingest.cuh"
#include "k_umma_image.cuh"
#include "k_step_fused.cuh"
#include "k_gemm_umma.cuh"
#include "k_layerwise.cuh"
#include "k_mesh.cuh"
#include "k_eval.cuh"
#include "k_assoc.cuh"
#include "k_hull.cuh"
#include "k_render.cuh"
#include "k_track.cuh"
#include "k_ba.cuh"
#include "k_track_lw.cuh"
#include "k_track_fused.cuh"
#include "k_reloc.cuh"

struct vmb_handle {
  int device, max_obj, H, nfreq;
  int n_sm;
  VmbLayout L;
  // Scratch of the entry points: device buffers that grow on demand and never move once a captured graph holds them
  // (DeviceBuffer), freed with the handle.
  DeviceBuffer<int> d_counts;          // [max_obj][4]
  DeviceBuffer<int> d_img_index;       // [P] param index -> half index inside the fp16 image (or -1)
  DeviceBuffer<unsigned int> d_ticket; // last-block ticket of the fused AdamW (device step counter mode)
  DeviceBuffer<unsigned int> d_smax;   // [max_obj] sampler: per-object max sampled depth (order-preserving key)
  DeviceBuffer<float> d_partials;      // fused step: [(max_obj + n_sm)][stride] per-(CTA, object) gradient partials (allocated on first use)
  DeviceBuffer<unsigned int> d_finish_sync; // fused step: finish sync words + per-object readiness counts and skip flags (uf::SY_*)
  DeviceBuffer<float2> d_bc;           // AdamW bias corrections per step number for (bc_b1, bc_b2), built on the host in double precision
  double bc_b1 = -1.0, bc_b2 = -1.0;
  int img_halves = 0;
  bool umma_ok = false;   // hidden 32: fused wgmma kernel + its pre-arranged fp16 image
  bool lw_ok = false;     // hidden 64/128/256: layer-wise wgmma GEMM path + row-major fp16 image
  lw::Workspace ws;       // training-step activations (may be baked into a captured graph)
  lw::Workspace ws_fwd;   // forward-only queries (vmb_forward): separate, so eval_points never moves the step's buffers
  mesh::Workspace ws_mesh;// marching cubes / unprojection scratch (grow-only)
  eval3d::Workspace ws_eval;// box crop / surface sampling / nearest-neighbour scratch (grow-only)
  assoc::Workspace ws_assoc;// ScanNet association scratch (grow-only)
  hull::Workspace ws_hull;  // convex hull / minimum-volume box scratch (grow-only)
  render::Workspace ws_render;// view rendering: source table, entry sort / scan scratch (grow-only)
  lw::TrackWorkspace ws_track;// layer-wise tracking step: its own, so a tracking capture never pins the mapping step's
  lw::TrackWorkspace ws_ba;   // layer-wise bundle-adjustment step: likewise (and tracking never moves a BA capture's)
  lw::JointWorkspace ws_joint;// joint map-and-pose step: world points and pose terms (the activations are the step's ws)
  tf::Workspace ws_tf;        // fused hidden-32 tracking step: per-ray rows before K10's tile sums (BA writes its rows)
  rl::Workspace ws_reloc;     // relocalisation scoring: per-(hypothesis, ray) loss terms before K10's tile sums
  std::string err;
};

static thread_local std::string g_err;

static int fail(vmb_handle* h, int code, const std::string& msg) {
  if (h) h->err = msg;
  g_err = msg;
  return code;
}
#define CUDA_TRY(h, expr)                                                                  \
  do {                                                                                     \
    cudaError_t e_ = (expr);                                                               \
    if (e_ != cudaSuccess)                                                                 \
      return fail(h, VMB_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));      \
  } while (0)

// points per tile (TP) of the CUDA-core fp32 network (NetTile) for hidden size H: K1 fp32, K10 and K11
static constexpr int fp32_tile(int H) { return H == 32 ? 128 : (H == 256 ? 32 : 64); }

template <int H, int TP>
static int launch_fp32(vmb_handle* h, const StepParams& sp, long long n_tiles_x, cudaStream_t st) {
  const size_t smem = NetTile<H, TP>::smem(h->L, VMB_NDIRS);    // then the kernel's sDp rows
  CUDA_TRY(h, (smem_limit_once<k_step_fp32<H, TP>>(h->device, (int)smem)));
  dim3 grid((unsigned)n_tiles_x, (unsigned)sp.B);
  k_step_fp32<H, TP><<<grid, 128, smem, st>>>(sp, h->L);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

static int dispatch_fp32(vmb_handle* h, const StepParams& sp, cudaStream_t st) {
  const int TP = fp32_tile(h->H);
  if (sp.S > TP) return fail(h, VMB_E_UNSUPPORTED, "fp32 step kernel: n_samples exceeds the tile size for this hidden size");
  const int nr = TP / sp.S;
  const long long tiles = ((long long)sp.R + nr - 1) / nr;
  if (tiles > 0x7fffffffLL || sp.B > 65535) return fail(h, VMB_E_ARG, "grid too large");
  switch (h->H) {
    case 32:  return launch_fp32<32, fp32_tile(32)>(h, sp, tiles, st);
    case 64:  return launch_fp32<64, fp32_tile(64)>(h, sp, tiles, st);
    case 128: return launch_fp32<128, fp32_tile(128)>(h, sp, tiles, st);
    case 256: return launch_fp32<256, fp32_tile(256)>(h, sp, tiles, st);
  }
  return fail(h, VMB_E_UNSUPPORTED, "unsupported hidden size");
}

extern "C" {

const char* vmb_version(void) { return "vmap_b200 0.1 (sm_90a)"; }

int vmb_param_count(int hidden, int n_freq) {
  if (hidden <= 0 || n_freq < 4 || n_freq > VMB_MAX_FREQ) return VMB_E_ARG;
  return vmb_make_layout(hidden, n_freq).P;
}
int vmb_param_stride(int hidden, int n_freq) {
  if (hidden <= 0 || n_freq < 4 || n_freq > VMB_MAX_FREQ) return VMB_E_ARG;
  return vmb_make_layout(hidden, n_freq).stride;
}
int vmb_param_offsets(int hidden, int n_freq, int* offsets, int* sizes) {
  if (hidden <= 0 || n_freq < 4 || n_freq > VMB_MAX_FREQ || !offsets || !sizes) return VMB_E_ARG;
  const VmbLayout L = vmb_make_layout(hidden, n_freq);
  const int H = hidden;
  const int off[VMB_N_TENSORS] = {L.o_Win, L.o_bin, L.o_Wm1, L.o_bm1, L.o_Wcat, L.o_bcat, L.o_Wm2, L.o_bm2,
                                  L.o_Wa, L.o_ba, L.o_Wcl, L.o_bcl, L.o_Woc, L.o_boc, L.o_B};
  const int sz[VMB_N_TENSORS] = {H * VMB_E1, H, H * H, H, H * (H + VMB_E1), H, H * H, H,
                                 H, 1, H * (H + L.e2), H, 3 * H, 3, VMB_NDIRS * 3};
  for (int i = 0; i < VMB_N_TENSORS; ++i) { offsets[i] = off[i]; sizes[i] = sz[i]; }
  return VMB_OK;
}
int vmb_image_bytes(int hidden, int n_freq) {
  if (hidden == 32 && n_freq == 6) return umma_image_bytes();
  if ((hidden == 64 || hidden == 128 || hidden == 256) && n_freq == 6) return (int)(2 * lw::img_halves(hidden));
  return 0;
}

const char* vmb_last_error(const vmb_handle* h) { return h ? h->err.c_str() : g_err.c_str(); }

int vmb_create(vmb_handle** out, int device, int max_obj, int hidden, int n_freq) {
  if (!out || max_obj <= 0) return fail(nullptr, VMB_E_ARG, "vmb_create: bad arguments");
  if (!(hidden == 32 || hidden == 64 || hidden == 128 || hidden == 256))
    return fail(nullptr, VMB_E_UNSUPPORTED, "vmb_create: hidden must be 32, 64, 128 or 256");
  if (n_freq < 4 || n_freq > VMB_MAX_FREQ) return fail(nullptr, VMB_E_ARG, "vmb_create: n_freq must be in [4,8]");
  CUDA_TRY(nullptr, cudaSetDevice(device));
  vmb_handle* h = new vmb_handle();
  h->device = device; h->max_obj = max_obj; h->H = hidden; h->nfreq = n_freq;
  h->n_sm = sm_count(device);
  h->L = vmb_make_layout(hidden, n_freq);
  cudaError_t e = h->d_counts.grow(sizeof(int) * 4 * max_obj, false);
  if (e == cudaSuccess) e = h->d_ticket.grow(sizeof(unsigned int), false);
  if (e == cudaSuccess) e = cudaMemset(h->d_ticket, 0, sizeof(unsigned int));
  if (e == cudaSuccess) e = h->d_smax.grow(sizeof(unsigned int) * (size_t)max_obj, false);
  if (e != cudaSuccess) { delete h; return fail(nullptr, VMB_E_NOMEM, cudaGetErrorString(e)); }
  if (hidden == 32 && n_freq == 6) {
    std::vector<int> idx(h->L.P);
    umma_fill_image_index(h->L, idx.data());
    h->img_halves = umma_image_bytes() / 2;
    e = h->d_img_index.grow(sizeof(int) * h->L.P, false);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_img_index, idx.data(), sizeof(int) * h->L.P, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { delete h; return fail(nullptr, VMB_E_CUDA, cudaGetErrorString(e)); }
    h->umma_ok = true;
  } else if ((hidden == 64 || hidden == 128 || hidden == 256) && n_freq == 6) {
    std::vector<int> idx(h->L.P);
    lw::fill_image_index(h->L, idx.data());
    h->img_halves = (int)lw::img_halves(hidden);
    e = h->d_img_index.grow(sizeof(int) * h->L.P, false);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_img_index, idx.data(), sizeof(int) * h->L.P, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { delete h; return fail(nullptr, VMB_E_CUDA, cudaGetErrorString(e)); }
    h->lw_ok = true;
  }
  *out = h;
  return VMB_OK;
}

void vmb_destroy(vmb_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  delete h;
}

int vmb_mask_counts(vmb_handle* h, int n_obj, int n_rays, const unsigned char* sem, long long sem_stride,
                    const unsigned char* mask_depth, long long mask_stride, int* out_counts, void* stream) {
  if (!h || n_obj <= 0 || n_rays <= 0 || !sem || !mask_depth || !out_counts)
    return fail(h, VMB_E_ARG, "vmb_mask_counts: bad arguments");
  k_mask_counts<<<n_obj, 256, 0, (cudaStream_t)stream>>>(n_rays, sem, sem_stride, mask_depth, mask_stride,
                                                         out_counts, nullptr);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// scalars exactly as torch.optim.adamw._single_tensor_adamw forms them (python doubles)
struct AdamScalars { float lr_wd, one_m_b1, b2, one_m_b2, step_size, bc2_sqrt; double lr, b1, b2d; };
static AdamScalars adam_scalars(float lr_f, float b1_f, float b2_f, float wd_f, int step) {
  AdamScalars q;
  const double lr = lr_f, b1 = b1_f, b2 = b2_f;
  q.lr = lr; q.b1 = b1; q.b2d = b2;
  q.lr_wd = (float)(1.0 - lr * (double)wd_f);
  q.one_m_b1 = (float)(1.0 - b1);
  q.b2 = (float)b2;
  q.one_m_b2 = (float)(1.0 - b2);
  const double t = (double)(step < 1 ? 1 : step);
  q.step_size = (float)(lr / (1.0 - std::pow(b1, t)));
  q.bc2_sqrt = (float)std::sqrt(1.0 - std::pow(b2, t));
  return q;
}

// scratch of the fused step kernel (gradient partial rows + finish sync words and skip flags): a fixed size, allocated
// on the first use and kept from then on, so later steps make no runtime call for it
static int fused_scratch(vmb_handle* h, cudaStream_t st) {
  if (h->d_finish_sync) return VMB_OK;
  const bool capturing = stream_capturing(st);
  const size_t rows = (size_t)fused_rows_needed(h->max_obj, h->n_sm);
  const size_t sync_bytes = sizeof(unsigned int) * (uf::SY_OBJ + 2 * (size_t)h->max_obj);
  cudaError_t e = h->d_partials.grow(rows * h->L.stride * sizeof(float), capturing);
  if (e == cudaSuccess) e = h->d_finish_sync.grow(sync_bytes, capturing);
  if (e == cudaSuccess) e = cudaMemset(h->d_finish_sync, 0, sync_bytes);
  if (e == cudaErrorStreamCaptureUnsupported)
    return fail(h, VMB_E_CUDA, "vmb_step: first fused step of a handle must run outside stream capture (scratch allocation)");
  if (e != cudaSuccess) return fail(h, VMB_E_NOMEM, cudaGetErrorString(e));
  return VMB_OK;
}

// Device table of AdamW's bias corrections (1 - b1^t, sqrt(1 - b2^t)) for t < BC_N, computed in double precision like
// torch.optim.adamw does; the kernels index it with the per-object device step number.  Rebuilt when the betas change
// (never during stream capture: a captured graph would keep using the pointer, whose CONTENT is what changes).
constexpr int BC_N = 20480;
static int ensure_bc_table(vmb_handle* h, double b1, double b2, cudaStream_t st) {
  if (h->d_bc && h->bc_b1 == b1 && h->bc_b2 == b2) return VMB_OK;
  if (stream_capturing(st))
    return fail(h, VMB_E_CUDA, "AdamW bias-correction table must be built outside stream capture (run one step eagerly first)");
  CUDA_TRY(h, h->d_bc.grow(sizeof(float2) * BC_N, false));
  std::vector<float2> tab(BC_N);
  for (int t = 0; t < BC_N; ++t) {
    const double tt = t < 1 ? 1.0 : (double)t;
    tab[t] = make_float2((float)(1.0 - std::pow(b1, tt)), (float)std::sqrt(1.0 - std::pow(b2, tt)));
  }
  CUDA_TRY(h, cudaStreamSynchronize(st));          // earlier launches may still read the old content
  CUDA_TRY(h, cudaMemcpy(h->d_bc, tab.data(), sizeof(float2) * BC_N, cudaMemcpyHostToDevice));
  h->bc_b1 = b1; h->bc_b2 = b2;
  return VMB_OK;
}

// scalar loss of a step for the paths that do not produce it inside their own kernels
__global__ void k_loss_sum(const float* __restrict__ loss_terms, int B, float* __restrict__ out) {
  float s = 0.f;
  for (int b = threadIdx.x; b < B; b += 32) s += loss_terms[b * 4 + 3];
  s = warp_sum(s);
  if (threadIdx.x == 0) *out = s;
}

static int launch_adamw(vmb_handle* h, int n_obj, float* params, float* grads, float* m, float* v, void* image,
                        const float* loss_terms, int* status, const AdamScalars& q, float eps, int zero_grads,
                        int* step_counter, cudaStream_t st, const float* loss_sum_src = nullptr, float* loss_sum = nullptr,
                        const float* grad_scale = nullptr) {
  if (h->L.stride < 1024) return fail(h, VMB_E_UNSUPPORTED, "vmb_adam: row pitch below one block");
  AdamParams p;
  memset(&p, 0, sizeof(p));
  p.n = (long long)n_obj * h->L.stride; p.stride = h->L.stride; p.P = h->L.P; p.B = n_obj;
  p.p = params; p.g = grads; p.m = m; p.v = v;
  p.image = (__half*)image; p.img_index = h->d_img_index; p.img_halves = h->img_halves;
  p.loss_terms = loss_terms; p.status = status; p.loss_sum_src = loss_sum_src; p.loss_sum = loss_sum; p.grad_scale = grad_scale;
  p.lr_wd = q.lr_wd; p.one_m_b1 = q.one_m_b1; p.b2 = q.b2; p.one_m_b2 = q.one_m_b2;
  p.step_counter = step_counter; p.ticket = h->d_ticket; p.lr = q.lr; p.b1 = q.b1; p.b2d = q.b2d;
  p.log_b1 = (float)std::log(q.b1); p.log_b2 = (float)std::log(q.b2d);
  if (step_counter) {
    const int rcb = ensure_bc_table(h, q.b1, q.b2d, st);
    if (rcb != VMB_OK) return rcb;
    p.bc_table = h->d_bc; p.bc_n = BC_N;
  }
  p.step_size = q.step_size; p.bc2_sqrt = q.bc2_sqrt;
  p.eps = eps;
  p.zero_grads = zero_grads;
  const long long n4 = p.n / 4;
  const int blocks = (int)((n4 + 255) / 256);
  k_adamw<<<blocks, 256, 0, st>>>(p);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// the argument checks of vmb_step (and of vmb_joint_step_lw, which takes the same struct) and the step's parameters
static int step_params(vmb_handle* h, const vmb_step_args* a, StepParams& sp, const std::string& who) {
  if (!h || !a) return fail(h, VMB_E_ARG, who + ": null argument");
  if (a->n_obj <= 0 || a->n_obj > h->max_obj || a->n_rays <= 0 || a->n_samples <= 0 || a->n_samples > 32)
    return fail(h, VMB_E_ARG, who + ": bad n_obj / n_rays / n_samples (1 <= S <= 32)");
  if (!a->pcs || !a->z_vals || !a->gt_depth || !a->gt_colour || !a->sem || !a->mask_depth || !a->params ||
      !a->scale || !a->loss_terms || (a->backward && !a->grads && !a->fuse_adam))
    return fail(h, VMB_E_ARG, who + ": missing tensor pointer");
  if (a->fuse_adam && (!a->backward || !a->exp_avg || !a->exp_avg_sq || (a->step < 1 && !a->step_counter)))
    return fail(h, VMB_E_ARG, who + ": fuse_adam needs backward = 1, exp_avg / exp_avg_sq and a step number");
  memset(&sp, 0, sizeof(sp));
  sp.B = a->n_obj; sp.R = a->n_rays; sp.S = a->n_samples;
  sp.pcs = a->pcs; sp.pcs_stride = a->pcs_stride;
  sp.z = a->z_vals; sp.z_stride = a->z_stride;
  sp.gt_depth = a->gt_depth; sp.gt_depth_stride = a->gt_depth_stride;
  sp.gt_colour = a->gt_colour; sp.gt_colour_stride = a->gt_colour_stride;
  sp.sem = a->sem; sp.sem_stride = a->sem_stride;
  sp.mask = a->mask_depth; sp.mask_stride = a->mask_stride;
  sp.params = a->params; sp.scale = a->scale; sp.grads = a->grads; sp.loss_terms = a->loss_terms;
  sp.r_depth = a->r_depth; sp.r_var = a->r_var; sp.r_colour = a->r_colour; sp.r_opacity = a->r_opacity;
  sp.cs = a->colour_scaling; sp.os = a->opacity_scaling; sp.backward = a->backward;
  return VMB_OK;
}

// K0 of the non-fused paths: the mask counts (computed here unless the caller passes them) and zeroed loss terms
static int step_counts(vmb_handle* h, const vmb_step_args* a, StepParams& sp, cudaStream_t st) {
  const int* counts = a->counts;
  if (!counts) {
    k_mask_counts<<<a->n_obj, 256, 0, st>>>(a->n_rays, a->sem, a->sem_stride, a->mask_depth, a->mask_stride,
                                            h->d_counts, a->loss_terms);
    CUDA_TRY(h, cudaGetLastError());
    counts = h->d_counts;
  } else {
    CUDA_TRY(h, cudaMemsetAsync(a->loss_terms, 0, sizeof(float) * 4 * a->n_obj, st));
  }
  sp.counts = counts;
  return VMB_OK;
}

// the fused hidden-32 step's extra arguments (vmb_step and vmb_joint_step_fused): scratch, counts and the fused AdamW
static int fused_extra(vmb_handle* h, const vmb_step_args* a, cudaStream_t st, FusedExtra& fx) {
  const int rc0 = fused_scratch(h, st);
  if (rc0 != VMB_OK) return rc0;
  memset(&fx, 0, sizeof(fx));
  fx.partials = h->d_partials; fx.finish_sync = h->d_finish_sync; fx.counts_in = a->counts; fx.counts_pub = h->d_counts;
  fx.fuse_adam = a->fuse_adam ? 1 : 0;
  if (a->fuse_adam) {
    const AdamScalars q = adam_scalars(a->lr, a->beta1, a->beta2, a->weight_decay, a->step);
    fx.p = const_cast<float*>(a->params); fx.m = a->exp_avg; fx.v = a->exp_avg_sq;
    fx.image_out = (__half*)const_cast<void*>(a->image); fx.img_index = h->d_img_index; fx.img_halves = h->img_halves;
    fx.step_counter = a->step_counter; fx.step_size = q.step_size; fx.bc2_sqrt = q.bc2_sqrt;
    fx.lr = q.lr; fx.b1d = q.b1; fx.b2d = q.b2d;
    fx.log_b1 = (float)std::log(q.b1); fx.log_b2 = (float)std::log(q.b2d);
    if (a->step_counter) {
      const int rcb = ensure_bc_table(h, q.b1, q.b2d, st);
      if (rcb != VMB_OK) return rcb;
      fx.bc_table = h->d_bc; fx.bc_n = BC_N;
    }
    fx.lr_wd = q.lr_wd; fx.one_m_b1 = q.one_m_b1; fx.b2 = q.b2; fx.one_m_b2 = q.one_m_b2; fx.eps = a->eps;
    fx.guard_loss = a->guard_loss; fx.status = a->status;
  }
  fx.loss_sum = a->loss_sum;
  return VMB_OK;
}

int vmb_step(vmb_handle* h, const vmb_step_args* a, void* stream) {
  StepParams sp;
  const int rc0 = step_params(h, a, sp, "vmb_step");
  if (rc0 != VMB_OK) return rc0;
  cudaStream_t st = (cudaStream_t)stream;
  int impl = a->impl;
  const bool umma_possible = h->umma_ok && a->image != nullptr;
  const bool lw_possible = h->lw_ok && a->image != nullptr;
  if (impl == VMB_IMPL_AUTO) impl = umma_possible ? VMB_IMPL_UMMA : (lw_possible ? VMB_IMPL_LAYERWISE : VMB_IMPL_FP32);
  struct EvGuard {      // records the optional K1 timing events around whichever kernel runs
    cudaEvent_t stop; cudaStream_t st;
    ~EvGuard() { if (stop) cudaEventRecord(stop, st); }
  };

  // ---- hidden 32: ONE launch (counts + step + ordered gradient reduction (+ AdamW)) ----------------------------
  if (impl == VMB_IMPL_UMMA) {
    if (!umma_possible) return fail(h, VMB_E_UNSUPPORTED, "vmb_step: tensor-core path needs hidden=32, n_freq=6 and an image");
    FusedExtra fx;
    const int rc0 = fused_extra(h, a, st, fx);
    if (rc0 != VMB_OK) return rc0;
    EvGuard evg{(cudaEvent_t)a->k1_stop_event, st};
    if (a->k1_start_event) cudaEventRecord((cudaEvent_t)a->k1_start_event, st);
    std::string err;
    const int rc = fused_launch_step(h->L, sp, fx, a->image, h->n_sm, st, err);
    if (rc != VMB_OK) return fail(h, rc, err);
    return VMB_OK;
  }

  // ---- other paths: K0 (mask counts) -> K1 -> [K2] ---------------------------------------------------------------
  const int rcc = step_counts(h, a, sp, st);
  if (rcc != VMB_OK) return rcc;
  if (a->backward && !a->grads) return fail(h, VMB_E_ARG, "vmb_step: this path needs the grads block");
  AdamScalars q;
  memset(&q, 0, sizeof(q));
  if (a->fuse_adam) q = adam_scalars(a->lr, a->beta1, a->beta2, a->weight_decay, a->step);
  int rc = VMB_OK;
  {
    EvGuard evg{(cudaEvent_t)a->k1_stop_event, st};
    if (a->k1_start_event) cudaEventRecord((cudaEvent_t)a->k1_start_event, st);
    if (impl == VMB_IMPL_LAYERWISE) {
      if (!lw_possible) return fail(h, VMB_E_UNSUPPORTED, "vmb_step: layer-wise path needs hidden 64/128/256, n_freq=6 and an image");
      std::string err;
      rc = lw::launch_step(h->ws, h->L, sp, a->image, st, err);
      if (rc != VMB_OK) return fail(h, rc, err);
    } else if (impl == VMB_IMPL_FP32) {
      rc = dispatch_fp32(h, sp, st);
      if (rc != VMB_OK) return rc;
    } else {
      return fail(h, VMB_E_ARG, "vmb_step: unknown impl");
    }
  }
  if (a->fuse_adam)                                   // the AdamW launch also writes the step's scalar loss
    return launch_adamw(h, a->n_obj, const_cast<float*>(a->params), a->grads, a->exp_avg, a->exp_avg_sq,
                        (h->umma_ok || h->lw_ok) ? const_cast<void*>(a->image) : nullptr,
                        a->guard_loss ? a->loss_terms : nullptr, a->status, q, a->eps, 1, a->step_counter, st,
                        a->loss_terms, a->loss_sum);
  if (a->loss_sum) { k_loss_sum<<<1, 32, 0, st>>>(a->loss_terms, a->n_obj, a->loss_sum); CUDA_TRY(h, cudaGetLastError()); }
  return VMB_OK;
}

int vmb_step_trace(vmb_handle* h, const vmb_step_args* a, unsigned long long* trace, long long trace_words, void* stream) {
  StepParams sp;
  const int rc0 = step_params(h, a, sp, "vmb_step_trace");
  if (rc0 != VMB_OK) return rc0;
  if (!h->umma_ok || !a->image || a->impl == VMB_IMPL_FP32 || a->impl == VMB_IMPL_LAYERWISE)
    return fail(h, VMB_E_UNSUPPORTED, "vmb_step_trace: the fused hidden-32 step only (hidden 32, n_freq 6, an image)");
  static_assert(VMB_TRACE_STRIDE == uf::TR_STRIDE, "trace row layout");
  const int max_grid = h->n_sm < uf::MAX_CTAS ? h->n_sm : uf::MAX_CTAS;
  if (!trace || trace_words < 2LL * max_grid * uf::TR_STRIDE)
    return fail(h, VMB_E_ARG, "vmb_step_trace: the trace needs 2 * min(#SMs, 192) rows of VMB_TRACE_STRIDE words");
  cudaStream_t st = (cudaStream_t)stream;
  FusedExtra fx;
  const int rc1 = fused_extra(h, a, st, fx);
  if (rc1 != VMB_OK) return rc1;
  std::string err;
  const int rc = fused_launch_step(h->L, sp, fx, a->image, h->n_sm, st, err, nullptr, trace);
  if (rc != VMB_OK) return fail(h, rc, err);
  return VMB_OK;
}

int vmb_forward(vmb_handle* h, const vmb_forward_args* a, void* stream) {
  if (!h || !a || a->n_obj <= 0 || a->n_obj > h->max_obj || a->n_points <= 0 || !a->points || !a->params ||
      !a->scale || !a->alpha || !a->colour)
    return fail(h, VMB_E_ARG, "vmb_forward: bad arguments");
  StepParams sp;
  memset(&sp, 0, sizeof(sp));
  if (a->n_points > 0x7fffffffLL) return fail(h, VMB_E_ARG, "vmb_forward: too many points per call");
  sp.B = a->n_obj; sp.R = (int)a->n_points; sp.S = 1;
  sp.pcs = a->points; sp.pcs_stride = a->points_stride;
  sp.params = a->params; sp.scale = a->scale;
  sp.fwd_only = 1;
  sp.out_alpha = a->alpha; sp.alpha_stride = a->alpha_stride;
  sp.out_colour = a->colour; sp.colour_stride = a->colour_stride;
  if (a->image && h->umma_ok) {
    std::string err;
    FusedExtra fx;
    memset(&fx, 0, sizeof(fx));
    const int rc = fused_launch_step(h->L, sp, fx, a->image, h->n_sm, (cudaStream_t)stream, err);
    if (rc != VMB_OK) return fail(h, rc, err);
    return VMB_OK;
  }
  if (a->image && h->lw_ok) {
    std::string err;
    const int rc = lw::launch_forward(h->ws_fwd, h->L, sp, a->image, (cudaStream_t)stream, err);
    if (rc != VMB_OK) return fail(h, rc, err);
    return VMB_OK;
  }
  return dispatch_fp32(h, sp, (cudaStream_t)stream);
}

int vmb_adam(vmb_handle* h, const vmb_adam_args* a, void* stream) {
  if (!h || !a || a->n_obj <= 0 || a->n_obj > h->max_obj || (a->step < 1 && !a->step_counter) || !a->params || !a->grads ||
      !a->exp_avg || !a->exp_avg_sq)
    return fail(h, VMB_E_ARG, "vmb_adam: bad arguments");
  if (a->image && !h->umma_ok && !h->lw_ok) return fail(h, VMB_E_UNSUPPORTED, "vmb_adam: no fp16 image for this hidden size");
  const AdamScalars q = adam_scalars(a->lr, a->beta1, a->beta2, a->weight_decay, a->step);
  return launch_adamw(h, a->n_obj, a->params, a->grads, a->exp_avg, a->exp_avg_sq, a->image, a->loss_terms, a->status, q,
                      a->eps, a->zero_grads, a->step_counter, (cudaStream_t)stream, nullptr, nullptr, a->grad_scale);
}

int vmb_build_image(vmb_handle* h, int n_obj, const float* params, void* image, void* stream) {
  if (!h || n_obj <= 0 || n_obj > h->max_obj || !params || !image) return fail(h, VMB_E_ARG, "vmb_build_image: bad arguments");
  if (!h->umma_ok && !h->lw_ok) return fail(h, VMB_E_UNSUPPORTED, "vmb_build_image: no fp16 image for this hidden size");
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(h, cudaMemsetAsync(image, 0, (size_t)n_obj * h->img_halves * 2, st));
  const long long n = (long long)n_obj * h->L.stride;
  k_build_image<<<(int)((n + 255) / 256), 256, 0, st>>>(n_obj, h->L.stride, h->L.P, params, (__half*)image,
                                                        h->d_img_index, h->img_halves);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_sample(vmb_handle* h, const vmb_sample_args* a, void* stream) {
  if (!h || !a || a->n_obj <= 0 || a->n_frames <= 0 || a->n_pix <= 0)
    return fail(h, VMB_E_ARG, "vmb_sample: bad arguments");
  if (a->n_bins_cam2surface < 1 || a->n_bins < 1 || a->n_bins_cam2surface + a->n_bins > 32)
    return fail(h, VMB_E_ARG, "vmb_sample: need 1 <= n1, n2 and n1+n2 <= 32");
  if ((long long)a->n_frames * a->n_pix >= (1LL << 29))      // Philox counter word 0 is ray * 8 + chunk (k_sampler.cuh)
    return fail(h, VMB_E_ARG, "vmb_sample: need n_frames * n_pix < 2^29 rays per object");
  const bool shared = a->store_rgbx != nullptr;
  if (shared && (!a->store_depth || !a->store_inst || !a->store_t_wc || !a->kf_slot || !a->kf_bbox || !a->obj_id ||
                 a->kf_stride <= 0))
    return fail(h, VMB_E_ARG, "vmb_sample: shared keyframe store needs depth/inst/t_wc/kf_slot/kf_bbox/obj_id/kf_stride");
  if (!shared && (!a->rgbs || !a->depths || !a->t_wc || !a->bbox))
    return fail(h, VMB_E_ARG, "vmb_sample: missing per-object keyframe pointer tables");
  if (!a->n_keyframes || !a->latest_kf || !a->rays_dir ||
      !a->bin_limits || !a->pcs || !a->z_vals || !a->gt_depth || !a->gt_colour || !a->sem || !a->mask_depth)
    return fail(h, VMB_E_ARG, "vmb_sample: missing tensor pointer");
  SampleParams p;
  memset(&p, 0, sizeof(p));
  p.B = a->n_obj; p.n_frames = a->n_frames; p.n_pix = a->n_pix; p.n1 = a->n_bins_cam2surface; p.n2 = a->n_bins;
  p.W = a->width; p.Hh = a->height; p.min_bound = a->min_bound; p.eps = a->surface_eps; p.oeps = a->stop_eps;
  p.rgbs = a->rgbs; p.depths = a->depths; p.t_wc = a->t_wc; p.bbox = a->bbox; p.n_kf = a->n_keyframes;
  p.latest = a->latest_kf; p.rays_dir = a->rays_dir; p.lim = a->bin_limits; p.seed = a->seed; p.offset = a->offset;
  p.inj_kf = a->inj_kf; p.inj_u_w = a->inj_u_w; p.inj_u_h = a->inj_u_h; p.inj_u_z = a->inj_u_z; p.inj_nrm = a->inj_nrm;
  p.pcs = a->pcs; p.z = a->z_vals; p.gt_depth = a->gt_depth; p.gt_colour = a->gt_colour; p.rgb_u8 = a->gt_rgb_u8;
  p.sem = a->sem; p.mask = a->mask_depth;
  p.st_rgbx = reinterpret_cast<const uchar4*>(a->store_rgbx); p.st_depth = a->store_depth; p.st_inst = a->store_inst;
  p.offset_dev = a->offset_dev;
  p.camera_frame = a->camera_frame; p.kf_out = a->kf_out;
  p.st_twc = a->store_t_wc; p.kf_slot = a->kf_slot; p.bbox_flat = a->kf_bbox; p.obj_id = a->obj_id; p.kf_stride = a->kf_stride;
  if (a->n_obj > h->max_obj) return fail(h, VMB_E_ARG, "vmb_sample: n_obj exceeds the handle's max_obj");
  const int N = a->n_frames * a->n_pix;
  // enough CTAs to fill the GPU a few times over, never more than one ray per thread needs
  int chunks = (N + 255) / 256;
  const int want = (8 * h->n_sm + a->n_obj - 1) / a->n_obj;
  if (chunks > want) chunks = want;
  if (chunks < 1) chunks = 1;
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(h, cudaMemsetAsync(h->d_smax, 0, sizeof(unsigned int) * a->n_obj, st));
  k_sample_gather<<<dim3(chunks, a->n_obj), 256, 0, st>>>(p, h->d_smax);
  const int smem_pts = 256 * (a->n_bins_cam2surface + a->n_bins) * 16;      // staged z + points of 256 rays
  CUDA_TRY(h, (smem_limit_once<k_sample_points<0, 0>>(h->device, 256 * 32 * 16)));
  CUDA_TRY(h, (smem_limit_once<k_sample_points<1, 9>>(h->device, 256 * 32 * 16)));
  CUDA_TRY(h, (smem_limit_once<k_sample_points<5, 9>>(h->device, 256 * 32 * 16)));
  const dim3 grid2(chunks, a->n_obj);
  if (a->n_bins_cam2surface == 1 && a->n_bins == 9)      k_sample_points<1, 9><<<grid2, 256, smem_pts, st>>>(p, h->d_smax);   // objects
  else if (a->n_bins_cam2surface == 5 && a->n_bins == 9) k_sample_points<5, 9><<<grid2, 256, smem_pts, st>>>(p, h->d_smax);   // background
  else                                                   k_sample_points<0, 0><<<grid2, 256, smem_pts, st>>>(p, h->d_smax);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// ---- K4: frame ingest (instance image -> per-instance boxes, shared-store write) ---------------------
int vmb_ingest_frame(vmb_handle* h, const vmb_ingest_args* a, void* stream) {
  if (!h || !a || a->width <= 0 || a->height <= 0 || a->max_id <= 0 || !a->inst || !a->stats || !a->bbox)
    return fail(h, VMB_E_ARG, "vmb_ingest_frame: bad arguments");
  if (a->bbox_scale < 0.f) return fail(h, VMB_E_ARG, "vmb_ingest_frame: bbox_scale must be >= 0 (utils.py:37)");
  if (a->bg_class && (!a->cls || a->n_class <= 0))
    return fail(h, VMB_E_ARG, "vmb_ingest_frame: bg_class needs the class image and n_class");
  const bool write = a->dst_inst != nullptr;
  if (write && ((a->rgb != nullptr) != (a->dst_rgbx != nullptr) || (a->depth != nullptr) != (a->dst_depth != nullptr)))
    return fail(h, VMB_E_ARG, "vmb_ingest_frame: rgb/depth sources and store destinations must come in pairs");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)a->width * a->height;
  const int blocks = 2 * h->n_sm;
  ing::k_ingest_init<<<(a->max_id + 255) / 256, 256, 0, st>>>(a->stats, a->max_id);
  ing::k_ingest_stats<<<blocks, 256, 0, st>>>(a->inst, a->cls, a->width, a->height, a->max_id, a->stats);
  ing::k_ingest_finalize<<<(a->max_id + 255) / 256, 256, 0, st>>>(a->stats, a->bbox, a->max_id, a->width, a->height,
                                                                 (float)(0.5 * (double)a->bbox_scale), a->min_extent,
                                                                 a->bg_class, a->n_class);
  if (write)
    ing::k_ingest_write<<<4 * h->n_sm, 256, 0, st>>>(a->inst, a->rgb, a->depth, a->stats, a->max_id, n,
                                                     reinterpret_cast<uchar4*>(a->dst_rgbx), a->dst_depth, a->dst_inst);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_store_relabel(vmb_handle* h, const vmb_relabel_args* a, void* stream) {
  if (!h || !a || a->width <= 0 || a->height <= 0 || a->max_id <= 0 || !a->labels || !a->assoc_bbox || !a->stats ||
      !a->bbox || !a->dst_inst)
    return fail(h, VMB_E_ARG, "vmb_store_relabel: bad arguments");
  if (a->assoc_max_id < 1 || a->assoc_max_id > a->max_id)
    return fail(h, VMB_E_ARG, "vmb_store_relabel: need 1 <= assoc_max_id <= max_id (labels must fit the store's tables)");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)a->width * a->height;
  const long long m = n > a->max_id ? n : a->max_id;
  long long g = (m + 255) / 256;
  if (g > 4 * h->n_sm) g = 4 * h->n_sm;
  ing::k_store_relabel<<<(unsigned)g, 256, 0, st>>>(a->labels, a->assoc_bbox, a->assoc_max_id, n, a->max_id,
                                                    a->dst_inst, a->stats, a->bbox);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// ---- K5: meshing (marching cubes, object-pixel unprojection) ---------------------------------------
static int mc_params(vmb_handle* h, const vmb_mc_args* a, mesh::McParams& q, const char* who) {
  if (!h || !a || !a->volume || a->nx < 2 || a->ny < 2 || a->nz < 2)
    return fail(h, VMB_E_ARG, std::string(who) + ": need a volume with nx, ny, nz >= 2");
  memset(&q, 0, sizeof(q));
  q.vol = a->volume; q.nx = a->nx; q.ny = a->ny; q.nz = a->nz; q.level = a->level;
  q.n = (long long)a->nx * a->ny * a->nz;
  if (3 * q.n >= 0x7fffffffLL || (long long)VMB_MC_MAX_TRI * q.n >= 0x7fffffffLL)
    return fail(h, VMB_E_ARG, std::string(who) + ": volume too large for int32 vertex / face indices");
  double A[9], det;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) { A[3 * r + c] = a->affine[4 * r + c]; q.M[3 * r + c] = a->affine[4 * r + c]; }
    q.o[r] = a->affine[4 * r + 3];
  }
  det = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
  if (!(std::fabs(det) > 0.0) || !std::isfinite(det)) return fail(h, VMB_E_ARG, std::string(who) + ": singular affine");
  // M^-T = cofactor(M) / det
  const double C[9] = {A[4] * A[8] - A[5] * A[7], A[5] * A[6] - A[3] * A[8], A[3] * A[7] - A[4] * A[6],
                       A[2] * A[7] - A[1] * A[8], A[0] * A[8] - A[2] * A[6], A[1] * A[6] - A[0] * A[7],
                       A[1] * A[5] - A[2] * A[4], A[2] * A[3] - A[0] * A[5], A[0] * A[4] - A[1] * A[3]};
  for (int i = 0; i < 9; ++i) q.Nt[i] = (float)(C[i] / det);
  return VMB_OK;
}

int vmb_mc_count(vmb_handle* h, const vmb_mc_args* a, void* stream) {
  mesh::McParams q;
  const int rc = mc_params(h, a, q, "vmb_mc_count");
  if (rc != VMB_OK) return rc;
  if (!a->totals) return fail(h, VMB_E_ARG, "vmb_mc_count: totals is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  mesh::Workspace& w = h->ws_mesh;
  const bool capturing = stream_capturing(st);
  const size_t n1 = (size_t)q.n + 1;
  CUDA_TRY(h, w.mc_bytes.grow(2 * n1 * sizeof(int) + 2 * (size_t)q.n, capturing));
  q.pt_scan = reinterpret_cast<int*>(w.mc_bytes.get());
  q.cell_scan = q.pt_scan + n1;
  q.pt_mask = reinterpret_cast<unsigned char*>(q.cell_scan + n1);
  q.cell_case = q.pt_mask + q.n;
  mesh::k_mc_count<<<mesh::blocks_for((long long)n1), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.scan(q.pt_scan, (long long)n1, capturing, st));
  CUDA_TRY(h, w.scan(q.cell_scan, (long long)n1, capturing, st));
  mesh::k_mc_totals<<<1, 1, 0, st>>>(q.pt_scan, q.cell_scan, q.n, a->totals);
  CUDA_TRY(h, cudaGetLastError());
  w.last = q;
  w.counted = true;
  return VMB_OK;
}

int vmb_mc_emit(vmb_handle* h, const vmb_mc_args* a, void* stream) {
  mesh::McParams q;
  const int rc = mc_params(h, a, q, "vmb_mc_emit");
  if (rc != VMB_OK) return rc;
  const mesh::McParams& c = h->ws_mesh.last;
  if (!h->ws_mesh.counted || c.vol != q.vol || c.nx != q.nx || c.ny != q.ny || c.nz != q.nz || c.level != q.level)
    return fail(h, VMB_E_ARG, "vmb_mc_emit: no matching vmb_mc_count on this handle (same volume, shape and level)");
  if ((a->max_vertices > 0 && !a->vertices) || (a->max_faces > 0 && !a->faces) || a->max_vertices < 0 || a->max_faces < 0)
    return fail(h, VMB_E_ARG, "vmb_mc_emit: output buffers missing for the given capacities");
  q.pt_scan = c.pt_scan; q.cell_scan = c.cell_scan; q.pt_mask = c.pt_mask; q.cell_case = c.cell_case;
  q.verts = a->vertices; q.normals = a->normals; q.faces = a->faces;
  q.max_verts = a->max_vertices; q.max_faces = a->max_faces;
  mesh::k_mc_emit<<<mesh::blocks_for(q.n), 256, 0, (cudaStream_t)stream>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_unproject(vmb_handle* h, const vmb_unproject_args* a, void* stream) {
  if (!h || !a || !a->count || a->width <= 0 || a->height <= 0 || a->n_keyframes < 0 || !(a->fx != 0.f) || !(a->fy != 0.f))
    return fail(h, VMB_E_ARG, "vmb_unproject: bad arguments");
  const bool store = a->store_depth != nullptr;
  if (store && (!a->store_inst || !a->store_t_wc || (a->n_keyframes > 0 && !a->kf_slot)))
    return fail(h, VMB_E_ARG, "vmb_unproject: shared keyframe store needs store_inst, store_t_wc and kf_slot");
  if (!store && (!a->rgbs || !a->depths || !a->t_wc))
    return fail(h, VMB_E_ARG, "vmb_unproject: per-object mode needs rgbs, depths and t_wc");
  if (a->max_points < 0 || (a->max_points > 0 && !a->points))
    return fail(h, VMB_E_ARG, "vmb_unproject: points missing for the given capacity");
  mesh::UnprojParams q;
  memset(&q, 0, sizeof(q));
  q.W = a->width; q.H = a->height; q.n_kf = a->n_keyframes;
  q.n = (long long)a->n_keyframes * a->width * a->height;
  if (q.n + 1 >= 0x7fffffffLL) return fail(h, VMB_E_ARG, "vmb_unproject: too many pixels for int32 indices");
  q.fx = a->fx; q.fy = a->fy; q.cx = a->cx; q.cy = a->cy;
  q.rgbs = reinterpret_cast<const uchar4*>(a->rgbs); q.depths = a->depths; q.t_wc = a->t_wc;
  q.st_depth = a->store_depth; q.st_inst = a->store_inst; q.st_twc = a->store_t_wc; q.kf_slot = a->kf_slot;
  q.obj_id = a->obj_id;
  q.out = a->points; q.max_points = a->points ? a->max_points : 0;
  mesh::Workspace& w = h->ws_mesh;
  cudaStream_t st = (cudaStream_t)stream;
  const bool capturing = stream_capturing(st);
  CUDA_TRY(h, w.up_scan.grow((size_t)(q.n + 1) * sizeof(int), capturing));
  q.scan = w.up_scan;
  mesh::k_unproj_flag<<<mesh::blocks_for(q.n + 1), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.scan(q.scan, q.n + 1, capturing, st));
  CUDA_TRY(h, cudaMemcpyAsync(a->count, q.scan + q.n, sizeof(int), cudaMemcpyDeviceToDevice, st));
  if (q.max_points > 0 && q.n > 0) {
    mesh::k_unproj_emit<<<mesh::blocks_for(q.n), 256, 0, st>>>(q);
    CUDA_TRY(h, cudaGetLastError());
  }
  return VMB_OK;
}

// ---- K6: 3-D reconstruction metrics (box crop, surface sampling, nearest neighbour) ---------------
static int clip_params(vmb_handle* h, const vmb_clip_args* a, eval3d::ClipParams& q, const char* who) {
  if (!h || !a || !a->vertices || !a->faces || a->n_vertices <= 0 || a->n_faces <= 0)
    return fail(h, VMB_E_ARG, std::string(who) + ": need a mesh with n_vertices, n_faces >= 1");
  if (a->n_vertices > 0x7fffffffLL || 7 * a->n_faces + 1 >= 0x7fffffffLL)
    return fail(h, VMB_E_ARG, std::string(who) + ": mesh too large for int32 indices");
  memset(&q, 0, sizeof(q));
  q.v = a->vertices; q.nv = a->n_vertices; q.f = a->faces; q.nf = a->n_faces;
  for (int j = 0; j < 3; ++j) {
    if (!(a->extent[j] >= 0.f)) return fail(h, VMB_E_ARG, std::string(who) + ": box extents must be >= 0");
    q.c[j] = a->center[j];
    q.half[j] = 0.5f * a->extent[j];
    for (int r = 0; r < 3; ++r) q.ax[j][r] = a->rotation[3 * r + j];
  }
  return VMB_OK;
}

int vmb_clip_count(vmb_handle* h, const vmb_clip_args* a, void* stream) {
  eval3d::ClipParams q;
  const int rc = clip_params(h, a, q, "vmb_clip_count");
  if (rc != VMB_OK) return rc;
  if (!a->count) return fail(h, VMB_E_ARG, "vmb_clip_count: count is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  eval3d::Workspace& w = h->ws_eval;
  const bool capturing = stream_capturing(st);
  CUDA_TRY(h, w.clip_scan.grow((size_t)(q.nf + 1) * sizeof(int), capturing));
  q.scan = w.clip_scan;
  eval3d::k_clip_count<<<eval3d::blocks_for(q.nf + 1, 128), 128, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.exclusive_sum(q.scan, q.nf + 1, capturing, st));
  CUDA_TRY(h, cudaMemcpyAsync(a->count, q.scan + q.nf, sizeof(int), cudaMemcpyDeviceToDevice, st));
  w.last = q;
  w.counted = true;
  return VMB_OK;
}

int vmb_clip_emit(vmb_handle* h, const vmb_clip_args* a, void* stream) {
  eval3d::ClipParams q;
  const int rc = clip_params(h, a, q, "vmb_clip_emit");
  if (rc != VMB_OK) return rc;
  const eval3d::ClipParams& c = h->ws_eval.last;
  if (!h->ws_eval.counted || c.v != q.v || c.nv != q.nv || c.f != q.f || c.nf != q.nf ||
      memcmp(c.c, q.c, sizeof(q.c)) || memcmp(c.ax, q.ax, sizeof(q.ax)) || memcmp(c.half, q.half, sizeof(q.half)))
    return fail(h, VMB_E_ARG, "vmb_clip_emit: no matching vmb_clip_count on this handle (same mesh and box)");
  if (a->max_triangles < 0 || (a->max_triangles > 0 && !a->triangles))
    return fail(h, VMB_E_ARG, "vmb_clip_emit: triangles missing for the given capacity");
  q.scan = c.scan; q.out = a->triangles; q.max_tri = a->max_triangles;
  eval3d::k_clip_emit<<<eval3d::blocks_for(q.nf, 128), 128, 0, (cudaStream_t)stream>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_surface_sample(vmb_handle* h, const vmb_surface_sample_args* a, void* stream) {
  if (!h || !a || !a->vertices || !a->faces || a->n_vertices <= 0 || a->n_faces <= 0 || a->n_points < 0)
    return fail(h, VMB_E_ARG, "vmb_surface_sample: need a mesh with n_vertices, n_faces >= 1 and n_points >= 0");
  if (a->n_vertices > 0x7fffffffLL || a->n_faces >= 0x7fffffffLL)
    return fail(h, VMB_E_ARG, "vmb_surface_sample: mesh too large for int32 indices");
  if (a->n_points > 0 && !a->points) return fail(h, VMB_E_ARG, "vmb_surface_sample: points is NULL");
  if (a->n_points == 0) return VMB_OK;
  eval3d::SampleSurfParams q;
  memset(&q, 0, sizeof(q));
  q.v = a->vertices; q.nv = a->n_vertices; q.f = a->faces; q.nf = a->n_faces;
  q.n = a->n_points; q.seed = a->seed; q.uniforms = a->uniforms; q.points = a->points; q.face_index = a->face_index;
  cudaStream_t st = (cudaStream_t)stream;
  eval3d::Workspace& w = h->ws_eval;
  const bool capturing = stream_capturing(st);
  CUDA_TRY(h, w.cum.grow((size_t)q.nf * sizeof(double) + sizeof(double), capturing));
  q.cum = w.cum;
  q.bad = reinterpret_cast<int*>(w.cum + q.nf);
  CUDA_TRY(h, cudaMemsetAsync(q.bad, 0, sizeof(int), st));
  eval3d::k_face_area<<<eval3d::blocks_for(q.nf, 256), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.inclusive_sum(q.cum, q.nf, capturing, st));
  double total = 0.0;
  int bad = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&total, q.cum + q.nf - 1, sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaMemcpyAsync(&bad, q.bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  if (bad) return fail(h, VMB_E_ARG, "vmb_surface_sample: a face index is outside [0, n_vertices)");
  if (!(total > 0.0) || !std::isfinite(total))
    return fail(h, VMB_E_ARG, "vmb_surface_sample: the mesh has no (finite) area");
  eval3d::k_sample_surface<<<eval3d::blocks_for(q.n, 256), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_nn_dist(vmb_handle* h, const vmb_nn_args* a, void* stream) {
  if (!h || !a || !a->ref || a->n_ref <= 0 || a->n_query < 0)
    return fail(h, VMB_E_ARG, "vmb_nn_dist: need n_ref >= 1 ref points and n_query >= 0");
  if (a->n_ref >= 0x7fffffffLL) return fail(h, VMB_E_ARG, "vmb_nn_dist: too many ref points for int32 indices");
  if (a->n_query > 0 && (!a->query || !a->dist)) return fail(h, VMB_E_ARG, "vmb_nn_dist: query / dist is NULL");
  if (a->n_query == 0) return VMB_OK;
  eval3d::NnParams q;
  memset(&q, 0, sizeof(q));
  q.ref = a->ref; q.n_ref = a->n_ref; q.query = a->query; q.n_q = a->n_query; q.dist = a->dist; q.index = a->index;
  q.max_cells = std::min<long long>(std::max<long long>(a->n_ref, 1), eval3d::EVAL_MAX_CELLS);
  // scratch: keys[6] (padded to 32 B) | Grid (padded to 64 B) | cell_start[max_cells+1] | pt_cell | pt_rank | sorted
  const size_t off_grid = 32, off_cells = 96;
  const size_t off_cell_pt = (off_cells + (size_t)(q.max_cells + 1) * sizeof(int) + 15) & ~(size_t)15;
  const size_t off_rank = off_cell_pt + (size_t)q.n_ref * sizeof(int);
  const size_t off_sorted = (off_rank + (size_t)q.n_ref * sizeof(int) + 15) & ~(size_t)15;
  const size_t need = off_sorted + (size_t)q.n_ref * sizeof(float4);
  eval3d::Workspace& w = h->ws_eval;
  cudaStream_t st = (cudaStream_t)stream;
  const bool capturing = stream_capturing(st);
  CUDA_TRY(h, w.nn.grow(need, capturing));
  q.keys = reinterpret_cast<unsigned int*>(w.nn.get());
  q.grid = reinterpret_cast<eval3d::Grid*>(w.nn + off_grid);
  q.cell_start = reinterpret_cast<int*>(w.nn + off_cells);
  q.pt_cell = reinterpret_cast<int*>(w.nn + off_cell_pt);
  q.pt_rank = reinterpret_cast<int*>(w.nn + off_rank);
  q.sorted = reinterpret_cast<float4*>(w.nn + off_sorted);
  CUDA_TRY(h, cudaMemsetAsync(q.keys, 0xff, 3 * sizeof(unsigned int), st));
  CUDA_TRY(h, cudaMemsetAsync(q.keys + 3, 0, 3 * sizeof(unsigned int), st));
  CUDA_TRY(h, cudaMemsetAsync(q.cell_start, 0, (size_t)(q.max_cells + 1) * sizeof(int), st));
  eval3d::k_nn_bbox<<<eval3d::blocks_for(q.n_ref, 256), 256, 0, st>>>(q);
  eval3d::k_nn_grid<<<1, 1, 0, st>>>(q);
  eval3d::k_nn_count<<<eval3d::blocks_for(q.n_ref, 256), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.exclusive_sum(q.cell_start, q.max_cells + 1, capturing, st));
  eval3d::k_nn_scatter<<<eval3d::blocks_for(q.n_ref, 256), 256, 0, st>>>(q);
  eval3d::k_nn_query<<<eval3d::blocks_for(q.n_q, 128), 128, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// ---- K7: ScanNet instance association (classify -> voxel -> finalize) ------------------------------
static int assoc_params(vmb_handle* h, const vmb_assoc_args* a, assoc::Params& q, bool capturing, const char* who) {
  if (!h || !a || a->width <= 0 || a->height <= 0 || !a->inst || !a->depth || !a->stats || !a->boxes)
    return fail(h, VMB_E_ARG, std::string(who) + ": bad arguments");
  if (a->max_id < 1 || a->max_id > 65536) return fail(h, VMB_E_ARG, std::string(who) + ": max_id must be in [1, 65536]");
  if ((long long)a->width * a->height >= 0x7fffffffLL) return fail(h, VMB_E_ARG, std::string(who) + ": image too large");
  if (a->bg_class && (!a->cls || a->n_class <= 0))
    return fail(h, VMB_E_ARG, std::string(who) + ": bg_class needs the class image and n_class");
  if (!(a->fx != 0.0) || !(a->fy != 0.0) || !(a->voxel_size > 0.0) || !(a->bbox_scale >= 0.0))
    return fail(h, VMB_E_ARG, std::string(who) + ": need fx, fy != 0, voxel_size > 0 and bbox_scale >= 0");
  if (a->n_pool < 0 || (a->n_pool > 0 && (!a->pool || !a->cloud_off || !a->cloud_cnt)) || a->n_pool >= 0x7fffffffLL)
    return fail(h, VMB_E_ARG, std::string(who) + ": pool needs cloud_off / cloud_cnt");
  memset(&q, 0, sizeof(q));
  q.W = a->width; q.H = a->height; q.max_id = a->max_id; q.n = (long long)a->width * a->height;
  q.inst = a->inst; q.cls = a->cls; q.depth = a->depth; q.bg_class = a->bg_class; q.n_class = a->n_class;
  q.fx = a->fx; q.fy = a->fy; q.cx = a->cx; q.cy = a->cy;
  for (int i = 0; i < 12; ++i) q.P[i] = a->camera_pose[i];
  q.min_pixels = a->min_pixels; q.voxel = a->voxel_size; q.half_voxel = a->voxel_size * 0.5;
  q.half_scale = 0.5 * a->bbox_scale;
  q.boxes = a->boxes; q.pool = a->pool; q.cloud_off = a->cloud_off; q.cloud_cnt = a->cloud_cnt;
  q.stats = a->stats;
  q.bound = a->n_pool + q.n;
  // scratch carving (pixel, id and element regions)
  assoc::Workspace& w = h->ws_assoc;
  const size_t n = (size_t)q.n, ni = (size_t)q.max_id + 1, nb = (size_t)q.bound;
  const size_t o_row = assoc::align16(n), o_k = o_row + assoc::align16(n), o_ko = o_k + 4 * n, o_v = o_ko + 4 * n,
               o_vo = o_v + 4 * n, pix_need = o_vo + 4 * n;
  CUDA_TRY(h, w.pix.grow(pix_need, capturing));
  q.flags = w.pix; q.rowok = w.pix + o_row;
  q.sel_key = (int*)(w.pix + o_k); q.sel_key_out = (int*)(w.pix + o_ko);
  q.sel_val = (int*)(w.pix + o_v); q.sel_val_out = (int*)(w.pix + o_vo);
  const size_t i_seg = assoc::align16(4 * ni), i_min = i_seg + assoc::align16(4 * ni), i_st = i_min + 24 * ni,
               i_ext = i_st + 16, ids_need = i_ext + 20 * ni;
  CUDA_TRY(h, w.ids.grow(ids_need, capturing));
  q.new_off = (int*)w.ids.get(); q.seg_off = (int*)(w.ids + i_seg);
  q.minb = (unsigned long long*)(w.ids + i_min); q.status = (int*)(w.ids + i_st);
  const size_t e_k = 24 * nb, e_ko = e_k + 8 * nb, e_i = e_ko + 8 * nb, e_io = e_i + 4 * nb,
               e_h = e_io + assoc::align16(4 * nb), el_need = e_h + 4 * (nb + 1);
  CUDA_TRY(h, w.el.grow(el_need, capturing));
  q.elem = (double*)w.el.get(); q.ekey = (unsigned long long*)(w.el + e_k); q.ekey_out = (unsigned long long*)(w.el + e_ko);
  q.eidx = (int*)(w.el + e_i); q.eidx_out = (int*)(w.el + e_io); q.head = (int*)(w.el + e_h);
  return VMB_OK;
}

static bool assoc_same(const assoc::Params& a, const assoc::Params& b) {
  return a.W == b.W && a.H == b.H && a.max_id == b.max_id && a.inst == b.inst && a.depth == b.depth &&
         a.stats == b.stats && a.boxes == b.boxes && a.pool == b.pool && a.bound == b.bound;
}

int vmb_assoc_classify(vmb_handle* h, const vmb_assoc_args* a, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool capturing = stream_capturing(st);
  assoc::Params q;
  const int rc = assoc_params(h, a, q, capturing, "vmb_assoc_classify");
  if (rc != VMB_OK) return rc;
  const unsigned gi = assoc::grid_for(q.max_id + 1, 256, 1 << 20), gp = assoc::grid_for(q.n, 256, 8 * h->n_sm);
  assoc::k_init<<<gi, 256, 0, st>>>(q);
  assoc::k_stats<<<gp, 256, 0, st>>>(q);
  assoc::k_erode_u<<<gp, 256, 0, st>>>(q);
  assoc::k_classify<<<gp, 256, 0, st>>>(q);
  assoc::k_decide<<<gi, 256, 0, st>>>(q);
  assoc::k_select<<<gp, 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  int end_bit = 1;
  while ((1 << end_bit) <= q.max_id) ++end_bit;
  assoc::Workspace& w = h->ws_assoc;
  size_t need = 0;
  CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(nullptr, need, q.sel_key, q.sel_key_out, q.sel_val, q.sel_val_out,
                                              (int)q.n, 0, end_bit, st));
  CUDA_TRY(h, w.cub_tmp.grow(need, capturing));
  CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(w.cub_tmp, need, q.sel_key, q.sel_key_out, q.sel_val, q.sel_val_out,
                                              (int)q.n, 0, end_bit, st));
  w.last = q;
  w.classified = true;
  return VMB_OK;
}

int vmb_assoc_voxel(vmb_handle* h, const vmb_assoc_args* a, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool capturing = stream_capturing(st);
  assoc::Params q;
  const int rc = assoc_params(h, a, q, capturing, "vmb_assoc_voxel");
  if (rc != VMB_OK) return rc;
  assoc::Workspace& w = h->ws_assoc;
  if (!w.classified || !assoc_same(w.last, q))
    return fail(h, VMB_E_ARG, "vmb_assoc_voxel: no matching vmb_assoc_classify on this handle");
  if (!a->cloud_out || a->max_cloud_out < q.bound)
    return fail(h, VMB_E_ARG, "vmb_assoc_voxel: cloud_out must hold n_pool + width * height points");
  const unsigned gi = assoc::grid_for(q.max_id + 1, 256, 1 << 20), ge = assoc::grid_for(q.bound, 256, 8 * h->n_sm);
  assoc::k_seg_len<<<gi, 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  size_t need = 0;
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(nullptr, need, q.seg_off, q.max_id + 1, st));
  CUDA_TRY(h, w.cub_tmp.grow(need, capturing));
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(w.cub_tmp, need, q.seg_off, q.max_id + 1, st));
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(w.cub_tmp, need, q.new_off, q.max_id + 1, st));
  assoc::k_elements<<<ge, 256, 0, st>>>(q);
  assoc::k_keys<<<ge, 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  need = 0;
  CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(nullptr, need, q.ekey, q.ekey_out, q.eidx, q.eidx_out, (int)q.bound, 0, 64, st));
  CUDA_TRY(h, w.cub_tmp.grow(need, capturing));
  CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(w.cub_tmp, need, q.ekey, q.ekey_out, q.eidx, q.eidx_out, (int)q.bound, 0, 64, st));
  assoc::k_heads<<<ge, 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  need = 0;
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(nullptr, need, q.head, (int)(q.bound + 1), st));
  CUDA_TRY(h, w.cub_tmp.grow(need, capturing));
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(w.cub_tmp, need, q.head, (int)(q.bound + 1), st));
  assoc::k_voxel_mean<<<ge, 256, 0, st>>>(q, a->cloud_out);
  CUDA_TRY(h, cudaGetLastError());
  int status = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&status, q.status, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  if (status) return fail(h, VMB_E_ARG, "vmb_assoc_voxel: a cloud spans more than 65536 voxels along an axis");
  return VMB_OK;
}

int vmb_assoc_finalize(vmb_handle* h, const vmb_assoc_args* a, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool capturing = stream_capturing(st);
  assoc::Params q;
  const int rc = assoc_params(h, a, q, capturing, "vmb_assoc_finalize");
  if (rc != VMB_OK) return rc;
  assoc::Workspace& w = h->ws_assoc;
  if (!w.classified || !assoc_same(w.last, q))
    return fail(h, VMB_E_ARG, "vmb_assoc_finalize: no matching vmb_assoc_classify on this handle");
  if (!a->final_label || !a->labels || !a->bbox) return fail(h, VMB_E_ARG, "vmb_assoc_finalize: bad arguments");
  assoc::FinParams f;
  memset(&f, 0, sizeof(f));
  f.W = q.W; f.H = q.H; f.max_id = q.max_id; f.n = q.n;
  f.inst = q.inst; f.depth = q.depth; f.stats = q.stats; f.flags = q.flags; f.final_label = a->final_label;
  f.labels = a->labels; f.bbox = a->bbox; f.half_scale = q.half_scale;
  f.ext = (int*)(w.ids + ((size_t)((unsigned char*)q.status - w.ids) + 16));
  const unsigned gi = assoc::grid_for(q.max_id + 1, 256, 1 << 20), gp = assoc::grid_for(q.n, 256, 8 * h->n_sm);
  assoc::k_fin_init<<<gi, 256, 0, st>>>(f);
  assoc::k_fin_label<<<gp, 256, 0, st>>>(f);
  assoc::k_fin_box<<<gi, 256, 0, st>>>(f);
  if (a->relabel) assoc::k_fin_relabel<<<gp, 256, 0, st>>>(f);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// ---- K8: convex hulls and minimum-volume boxes ----------------------------------------------------
static unsigned grid_of(long long n, int per, long long cap) {
  long long g = (n + per - 1) / per;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (unsigned)g;
}

int vmb_hull(vmb_handle* h, const vmb_hull_args* a, void* stream) {
  using namespace hull;
  if (!h || !a || a->n_points < 0 || (a->n_points > 0 && !a->points) || !a->set_size || a->size_stride < 1 ||
      a->n_sets < 1 || !a->is_vertex || !a->vertex_count || !a->status || !a->facets || !a->facet_count ||
      (a->vertices && !a->vertex_offset))
    return fail(h, VMB_E_ARG, "vmb_hull: bad arguments");
  if (a->n_points >= (1LL << 29)) return fail(h, VMB_E_ARG, "vmb_hull: too many points for int32 facet rows");
  const long long n = a->n_points;
  const int ns = a->n_sets;
  const long long fcap = facet_cap(n, ns);
  Params q;
  memset(&q, 0, sizeof(q));
  q.pts = a->points; q.n = n; q.set_size = a->set_size; q.size_stride = a->size_stride; q.n_sets = ns;
  q.is_vertex = a->is_vertex; q.vertex_count = a->vertex_count; q.status = a->status;
  q.facets = a->facets; q.facet_nbr = a->facet_nbr; q.facet_count = a->facet_count; q.fcap = fcap;
  // scratch: per-set ints | per-point bytes and ints | facet work regions
  const size_t si = align256(4 * (size_t)(ns + 1)), pb = align256((size_t)n + 1), pi = align256(4 * (size_t)n + 4),
               fi = align256(4 * (size_t)fcap);
  const size_t need = 11 * si + 256 + 2 * pb + 4 * pi + 12 * fi;
  Workspace& w = h->ws_hull;
  cudaStream_t st = (cudaStream_t)stream;
  const bool capturing = stream_capturing(st);
  CUDA_TRY(h, w.buf.grow(need, capturing));
  unsigned char* c = w.buf;
  auto take = [&](size_t bytes) { unsigned char* r = c; c += bytes; return r; };
  q.size = (int*)take(si); q.start = (int*)take(si);
  for (int k = 0; k < 3; ++k) q.cnt[k] = (int*)take(si);
  for (int k = 0; k < 2; ++k) q.off[k] = (int*)take(si);
  q.red = (int*)take(si); q.ntile = (int*)take(si); q.tile_start = (int*)take(si);
  int* vcount1 = (int*)take(si);
  q.n_sel = (int*)take(256);
  q.mark = take(pb); q.keep = take(pb);
  for (int k = 0; k < 2; ++k) q.list[k] = (int*)take(pi);
  q.start_at = (int*)take(pi); q.end_at = (int*)take(pi);
  q.fv = (int*)take(3 * fi); q.fn = (int*)take(3 * fi); q.fs = (int*)take(fi); q.vis = (int*)take(fi);
  q.fre = (int*)take(fi); q.hz = (int*)take(3 * fi);
  const int ni = (int)std::max<long long>(n, 1);
  size_t t1 = 0, t2 = 0, t3 = 0;
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(nullptr, t1, q.size, q.start, ns + 1, st));
  CUDA_TRY(h, cub::DeviceSelect::Flagged(nullptr, t2, q.list[0], q.keep, q.list[1], q.n_sel, ni, st));
  CUDA_TRY(h, cub::DeviceSelect::Flagged(nullptr, t3, thrust::counting_iterator<int>(0), q.is_vertex, q.list[1],
                                         q.n_sel, ni, st));
  CUDA_TRY(h, w.cub_tmp.grow(std::max(t1, std::max(t2, t3)), capturing));
  size_t tb = w.cub_tmp.bytes();
  const unsigned gs = grid_of(ns + 1, 256, 4096), gn = grid_of(n, 256, 8 * (long long)h->n_sm);
  k_sizes<<<gs, 256, 0, st>>>(q, q.cnt[0]);
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(w.cub_tmp, tb, q.size, q.start, ns + 1, st));
  k_init<<<gn, 256, 0, st>>>(q, q.cnt[0]);
  CUDA_TRY(h, cudaGetLastError());
  const int* cnt = q.cnt[0];
  const int* prev = nullptr;
  const int* off = q.start;
  const int* list = q.list[0];
  if (n > TILE)
    for (int r = 0; r < ROUNDS; ++r) {
      int* nxt = q.cnt[(r + 1) % 3];
      int* off_n = q.off[r % 2];
      int* list_n = q.list[(r + 1) % 2];
      k_tiles<<<gs, 256, 0, st>>>(q, cnt, prev, q.red, nxt);
      CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(w.cub_tmp, tb, q.ntile, q.tile_start, ns + 1, st));
      k_tile<<<(unsigned)max_tiles(n, ns), NT, 0, st>>>(q, cnt, off, list, q.red, nxt);
      k_keep<<<gn, 256, 0, st>>>(q, off, list);
      CUDA_TRY(h, cudaGetLastError());
      CUDA_TRY(h, cub::DeviceSelect::Flagged(w.cub_tmp, tb, list, q.keep, list_n, q.n_sel, ni, st));
      CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(w.cub_tmp, tb, nxt, off_n, ns + 1, st));
      prev = cnt; cnt = nxt; off = off_n; list = list_n;
    }
  k_final<<<ns, NT, 0, st>>>(q, cnt, off, list);
  CUDA_TRY(h, cudaGetLastError());
  if (a->vertex_offset) {
    CUDA_TRY(h, cudaMemsetAsync(vcount1 + ns, 0, sizeof(int), st));
    CUDA_TRY(h, cudaMemcpyAsync(vcount1, a->vertex_count, sizeof(int) * ns, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(w.cub_tmp, tb, vcount1, a->vertex_offset, ns + 1, st));
  }
  if (a->vertices && n > 0)
    CUDA_TRY(h, cub::DeviceSelect::Flagged(w.cub_tmp, tb, thrust::counting_iterator<int>(0), q.is_vertex,
                                           a->vertices, q.n_sel, ni, st));
  return VMB_OK;
}

int vmb_obb_minvol(vmb_handle* h, const vmb_obb_args* a, void* stream) {
  using namespace hull;
  if (!h || !a || !a->points || !a->facets || !a->facet_nbr || !a->facet_count || !a->vertices || !a->vertex_count ||
      !a->status || !a->box || !a->box_status || a->max_facets < 0)
    return fail(h, VMB_E_ARG, "vmb_obb_minvol: bad arguments");
  const long long cap = std::max<long long>(a->max_facets, 1);
  Workspace& w = h->ws_hull;
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(h, w.obb.grow(15 * sizeof(double) * (size_t)cap, stream_capturing(st)));
  ObbParams q;
  q.pts = a->points; q.facets = a->facets; q.facet_nbr = a->facet_nbr; q.facet_count = a->facet_count;
  q.vertices = a->vertices; q.vertex_count = a->vertex_count; q.status = a->status;
  q.box = a->box; q.box_status = a->box_status;
  q.nr = w.obb; q.nu = w.obb + 3 * cap; q.res = w.obb + 6 * cap;
  k_obb_normals<<<grid_of(cap, 256, 8 * (long long)h->n_sm), 256, 0, st>>>(q);
  k_obb_eval<<<grid_of(cap, 1, 8 * (long long)h->n_sm), NT, 0, st>>>(q);
  k_obb_pick<<<1, NT, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// ---- K9: view rendering (ray / box cull, sample emission, compositing) -----------------------------
static bool finite_all(const double* v, int n) {
  for (int i = 0; i < n; ++i)
    if (!std::isfinite(v[i])) return false;
  return true;
}

// checks shared by the three render entry points; fills the geometry part of q and uploads the source table
static int render_params(vmb_handle* h, const vmb_render_args* a, render::Params& q, bool capturing, const char* who) {
  const std::string w(who);
  if (!h || !a) return fail(h, VMB_E_ARG, w + ": null argument");
  if (a->width <= 0 || a->height <= 0) return fail(h, VMB_E_ARG, w + ": width and height must be >= 1");
  if (a->n_src < 1 || a->n_src > VMB_RENDER_MAX_SRC) return fail(h, VMB_E_ARG, w + ": n_src must be in [1, 1024]");
  if (a->n_coarse < 1 || a->n_fine < 0) return fail(h, VMB_E_ARG, w + ": need n_coarse >= 1 and n_fine >= 0");
  if (a->pass != 0 && a->pass != 1) return fail(h, VMB_E_ARG, w + ": pass must be 0 or 1");
  if (a->pass == 1 && a->n_fine == 0) return fail(h, VMB_E_ARG, w + ": pass 1 needs n_fine >= 1");
  const double intr[4] = {a->fx, a->fy, a->cx, a->cy};
  if (!finite_all(intr, 4) || a->fx == 0.0 || a->fy == 0.0)
    return fail(h, VMB_E_ARG, w + ": intrinsics must be finite with fx, fy != 0");
  if (!finite_all(a->t_wc, 12)) return fail(h, VMB_E_ARG, w + ": non-finite pose");
  if (!std::isfinite(a->near_depth) || !(a->near_depth >= 0.0) || !(a->far_depth > a->near_depth) ||
      std::isnan(a->far_depth))
    return fail(h, VMB_E_ARG, w + ": need 0 <= near < far");
  if (a->n_fine > 0 && !(std::isfinite(a->surface_eps) && a->surface_eps > 0.0))
    return fail(h, VMB_E_ARG, w + ": surface_eps must be finite and > 0");
  const long long n_pix = (long long)a->width * a->height;
  if (a->n_rays < 1 || a->ray0 < 0 || a->ray0 + a->n_rays > n_pix)
    return fail(h, VMB_E_ARG, w + ": rays [ray0, ray0 + n_rays) must lie inside the view");
  const long long n_e = (long long)a->n_rays * VMB_RENDER_MAX_HITS;
  if (n_e * std::max(a->n_coarse, a->n_fine) >= 0x7fffffffLL)
    return fail(h, VMB_E_ARG, w + ": n_rays * 16 * max(n_coarse, n_fine) exceeds int32 sample indices");
  if (!a->boxes || !a->obj_id) return fail(h, VMB_E_ARG, w + ": boxes / obj_id missing");
  for (int s = 0; s < a->n_src; ++s) {
    const double* b = a->boxes + (size_t)s * VMB_RENDER_BOX;
    if (!finite_all(b, VMB_RENDER_BOX)) return fail(h, VMB_E_ARG, w + ": non-finite box");
    if (!(b[12] > 0.0 && b[13] > 0.0 && b[14] > 0.0)) return fail(h, VMB_E_ARG, w + ": box half-extents must be > 0");
  }
  if (!a->hit_src || !a->hit_t || !a->hit_count) return fail(h, VMB_E_ARG, w + ": hit table missing");
  memset(&q, 0, sizeof(q));
  q.W = a->width; q.H = a->height;
  q.fx = a->fx; q.fy = a->fy; q.cx = a->cx; q.cy = a->cy;
  for (int i = 0; i < 12; ++i) q.T[i] = a->t_wc[i];
  q.near_ = a->near_depth; q.far_ = a->far_depth; q.eps = a->surface_eps;
  q.n_src = a->n_src; q.ray0 = a->ray0; q.n_rays = a->n_rays;
  q.n_coarse = a->n_coarse; q.n_fine = a->n_fine; q.pass = a->pass;
  q.hit_src = a->hit_src; q.hit_t = a->hit_t; q.hit_count = a->hit_count;
  q.overflow = a->overflow; q.src_total = a->src_total; q.zstar = a->zstar; q.surf = a->surf;
  render::Workspace& ws = h->ws_render;
  CUDA_TRY(h, ws.boxes.grow((size_t)a->n_src * VMB_RENDER_BOX * sizeof(double), capturing));
  CUDA_TRY(h, ws.obj_id.grow((size_t)a->n_src * sizeof(int), capturing));
  q.boxes = ws.boxes; q.obj_id = ws.obj_id;
  return VMB_OK;
}

static int render_upload(vmb_handle* h, const vmb_render_args* a, cudaStream_t st) {
  render::Workspace& ws = h->ws_render;
  CUDA_TRY(h, cudaMemcpyAsync(ws.boxes, a->boxes, (size_t)a->n_src * VMB_RENDER_BOX * sizeof(double),
                              cudaMemcpyHostToDevice, st));
  CUDA_TRY(h, cudaMemcpyAsync(ws.obj_id, a->obj_id, (size_t)a->n_src * sizeof(int), cudaMemcpyHostToDevice, st));
  return VMB_OK;
}

static bool render_same(const render::Params& x, const render::Params& y) {
  return x.pass == y.pass && x.ray0 == y.ray0 && x.n_rays == y.n_rays && x.n_src == y.n_src && x.W == y.W &&
         x.H == y.H && x.n_coarse == y.n_coarse && x.n_fine == y.n_fine && x.hit_src == y.hit_src &&
         x.hit_t == y.hit_t && x.hit_count == y.hit_count && x.zstar == y.zstar && x.eps == y.eps &&
         x.fx == y.fx && x.fy == y.fy && x.cx == y.cx && x.cy == y.cy && !memcmp(x.T, y.T, sizeof(x.T));
}

int vmb_render_count(vmb_handle* h, const vmb_render_args* a, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool capturing = stream_capturing(st);
  render::Params q;
  int rc = render_params(h, a, q, capturing, "vmb_render_count");
  if (rc != VMB_OK) return rc;
  if (!a->overflow || !a->src_total) return fail(h, VMB_E_ARG, "vmb_render_count: overflow / src_total missing");
  if (a->pass == 1 && !a->zstar) return fail(h, VMB_E_ARG, "vmb_render_count: pass 1 needs zstar");
  if ((rc = render_upload(h, a, st)) != VMB_OK) return rc;
  render::Workspace& ws = h->ws_render;
  const long long n_e = (long long)q.n_rays * VMB_RENDER_MAX_HITS;
  const size_t n1 = (size_t)n_e + 1;
  CUDA_TRY(h, ws.ints.grow(7 * n1 * sizeof(int), capturing));
  q.keys = ws.ints; q.keys_alt = q.keys + n1; q.vals = q.keys_alt + n1; q.vals_alt = q.vals + n1;
  q.cnt = q.vals_alt + n1;
  int* scan = q.cnt + n1;
  q.wbase = scan + n1;
  if (q.pass == 0) {
    CUDA_TRY(h, cudaMemsetAsync(q.overflow, 0, sizeof(int), st));
    render::k_cull<<<render::blocks_for(q.n_rays, 128), 128, 0, st>>>(q);
    CUDA_TRY(h, cudaGetLastError());
  }
  CUDA_TRY(h, cudaMemsetAsync(q.src_total, 0, (size_t)q.n_src * sizeof(int), st));
  render::k_entry_counts<<<render::blocks_for(n_e + 1, 256), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  // stable sort of the entries by source: the source-major sample order (ties keep ray order)
  size_t need = 0, need_scan = 0;
  CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(nullptr, need, q.keys, q.keys_alt, q.vals, q.vals_alt, (int)n_e, 0, 11, st));
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(nullptr, need_scan, scan, (int)n1, st));
  CUDA_TRY(h, ws.cub_tmp.grow(std::max(need, need_scan), capturing));
  CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(ws.cub_tmp, need, q.keys, q.keys_alt, q.vals, q.vals_alt, (int)n_e, 0, 11, st));
  render::k_gather_counts<<<render::blocks_for(n_e + 1, 256), 256, 0, st>>>(q, q.vals_alt, q.cnt, scan);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(ws.cub_tmp, need_scan, scan, (int)n1, st));
  render::k_scatter_base<<<render::blocks_for(n_e, 256), 256, 0, st>>>(q, q.vals_alt, scan, q.wbase);
  CUDA_TRY(h, cudaGetLastError());
  ws.last = q;
  ws.counted = true;
  return VMB_OK;
}

int vmb_render_emit(vmb_handle* h, const vmb_render_args* a, void* stream) {
  render::Params q;
  const int rc = render_params(h, a, q, stream_capturing((cudaStream_t)stream), "vmb_render_emit");
  if (rc != VMB_OK) return rc;
  render::Workspace& ws = h->ws_render;
  if (!ws.counted || !render_same(q, ws.last))
    return fail(h, VMB_E_ARG, "vmb_render_emit: no matching vmb_render_count on this handle (same rays, pass and tables)");
  if (!a->points || !a->z || !a->base) return fail(h, VMB_E_ARG, "vmb_render_emit: points / z / base missing");
  q.wbase = ws.last.wbase;
  q.points = a->points; q.z = a->z; q.base = a->base;
  const long long n_e = (long long)q.n_rays * VMB_RENDER_MAX_HITS;
  render::k_emit<<<render::blocks_for(n_e, 128), 128, 0, (cudaStream_t)stream>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_render_composite(vmb_handle* h, const vmb_render_args* a, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  render::Params q;
  int rc = render_params(h, a, q, stream_capturing(st), "vmb_render_composite");
  if (rc != VMB_OK) return rc;
  const bool images = a->pass == 1 || a->n_fine == 0;
  if (!a->z_coarse || !a->alpha_coarse || !a->colour_coarse || !a->base_coarse)
    return fail(h, VMB_E_ARG, "vmb_render_composite: coarse samples missing");
  if (a->pass == 1 && (!a->z_fine || !a->alpha_fine || !a->colour_fine || !a->base_fine))
    return fail(h, VMB_E_ARG, "vmb_render_composite: fine samples missing");
  if (!a->zstar || (a->pass == 0 && !a->surf)) return fail(h, VMB_E_ARG, "vmb_render_composite: zstar / surf missing");
  if (images && (!a->depth || !a->colour || !a->opacity || !a->instance))
    return fail(h, VMB_E_ARG, "vmb_render_composite: output images missing");
  if ((rc = render_upload(h, a, st)) != VMB_OK) return rc;
  q.z_c = a->z_coarse; q.alpha_c = a->alpha_coarse; q.colour_c = a->colour_coarse; q.base_c = a->base_coarse;
  q.z_f = a->z_fine; q.alpha_f = a->alpha_fine; q.colour_f = a->colour_fine; q.base_f = a->base_fine;
  q.depth = a->depth; q.colour = a->colour; q.opacity = a->opacity; q.instance = a->instance;
  render::k_composite<<<render::blocks_for(q.n_rays, 128), 128, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// ---- test hook for the generic wgmma GEMM of the layer-wise (wide model) path --------
// a_mn / b_mn = 0: operand stored [M or N rows][ld] with K contiguous; 1: stored [K rows][ld] with M or N contiguous.
// epi 0: out16 = relu(acc*scale + bias) (fp16);  epi 2: out32 (=|+=) acc*scale;  epi 3: atomicAdd(out32, acc*scale)
int vmb_debug_gemm(int a_mn, int b_mn, int epi, int M, int N, int K1, int K2, const void* a1, long long a1_ld,
                   const void* a2, long long a2_ld, const void* b, long long b_ld, const float* bias, void* out16, int ldo,
                   float* out32, int ld32, int accumulate, int ksplit, float scale, void* stream) {
  using namespace lw;
  const int K = K1 + K2;
  const bool ws = (epi & 16) != 0;             // +16: weight-stationary kernel (no fallback: the test wants THAT kernel)
  epi &= 15;
  Operand A1{a1, a_mn ? K1 : M, a_mn ? M : K1, a1_ld};
  Operand A2{a2, a_mn ? K2 : M, a_mn ? M : K2, a2_ld};
  Operand B{b, b_mn ? K : N, b_mn ? N : K, b_ld};
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.M = M; g.N = N; g.K1 = K1; g.K2 = K2; g.ksplit = ksplit; g.bias = bias; g.out16 = (__half*)out16; g.ldo = ldo;
  g.out32 = out32; g.ld32 = ld32; g.accumulate = accumulate; g.gdst = out32; g.ldgd = ld32; g.ldgn = 1; g.n_lo = 0; g.n_valid = N; g.ones_col = -1;
  g.scale = scale;
  const int mt = (M + BM - 1) / BM, nt = (N + BN - 1) / BN, z = ksplit > 0 ? (K + ksplit - 1) / ksplit : 1;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaErrorInvalidValue;
  if (ws) {
    if (a_mn == 0 && b_mn == 0 && epi == 0) e = launch_gemm_ws<0, EPI_RELU_F16>(A1, A2, B, g, mt, st);
    else if (a_mn == 0 && b_mn == 0 && epi == 2) e = launch_gemm_ws<0, EPI_F32>(A1, A2, B, g, mt, st);
    else if (a_mn == 0 && b_mn == 1 && epi == 2) e = launch_gemm_ws<1, EPI_F32>(A1, A2, B, g, mt, st);
  } else
  if (a_mn == 0 && b_mn == 0 && epi == 0) e = launch_gemm<0, 0, EPI_RELU_F16>(A1, A2, B, g, mt, nt, z, st);
  else if (a_mn == 0 && b_mn == 0 && epi == 2) e = launch_gemm<0, 0, EPI_F32>(A1, A2, B, g, mt, nt, z, st);
  else if (a_mn == 0 && b_mn == 1 && epi == 2) e = launch_gemm<0, 1, EPI_F32>(A1, A2, B, g, mt, nt, z, st);
  else if (a_mn == 1 && b_mn == 1 && epi == 3) e = launch_gemm<1, 1, EPI_ATOMIC>(A1, A2, B, g, mt, nt, z, st);
  if (e != cudaSuccess) return fail(nullptr, VMB_E_CUDA, std::string("vmb_debug_gemm: ") + cudaGetErrorString(e));
  return VMB_OK;
}

}  // extern "C"

// ---- K10 / K11, their layer-wise path and their fused hidden-32 path: one host path for the six step entry points ----
// which network runs the step: K10 / K11 on CUDA cores, the layer-wise wgmma GEMMs (hidden 64/128/256) or the fused
// hidden-32 wgmma tile
enum PosePath { POSE_FP32 = 0, POSE_LW = 1, POSE_FUSED = 2 };

template <int H, int TP, bool BA>
static int launch_pose(vmb_handle* h, const TrackParams& tp, const BaRays& x, int tiles, cudaStream_t st) {
  const size_t smem = NetTile<H, TP>::smem(h->L, 0);
  const dim3 grid((unsigned)tiles, (unsigned)tp.B);
  if constexpr (BA) {
    CUDA_TRY(h, (smem_limit_once<k_ba_step<H, TP>>(h->device, (int)smem)));
    k_ba_step<H, TP><<<grid, 128, smem, st>>>(tp, h->L, x);
  } else {
    CUDA_TRY(h, (smem_limit_once<k_track_step<H, TP>>(h->device, (int)smem)));
    k_track_step<H, TP><<<grid, 128, smem, st>>>(tp, h->L);
  }
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// the checks shared by every tracking (vmb_track_args) and bundle-adjustment (vmb_ba_args) entry point
template <class Args>
static int pose_args_ok(vmb_handle* h, const Args* a, const char* who) {
  if (!a) return fail(h, VMB_E_ARG, std::string(who) + ": null argument");
  if (a->n_groups < 1 || a->n_groups > VMB_TRACK_MAX_GROUPS)
    return fail(h, VMB_E_ARG, std::string(who) + ": n_groups must be in [1, 8]");
  if (a->n_iter < 1 || a->iter < 1 || a->iter > a->n_iter)
    return fail(h, VMB_E_ARG, std::string(who) + ": need n_iter >= 1 and 1 <= iter <= n_iter");
  if constexpr (std::is_same_v<Args, vmb_ba_args>) {
    if (!a->poses || a->n_poses < 1) return fail(h, VMB_E_ARG, std::string(who) + ": need a pose table");
  } else {
    if (!a->pose) return fail(h, VMB_E_ARG, std::string(who) + ": pose is NULL");
  }
  return VMB_OK;
}

static int ba_group_ok(const vmb_ba_group& g) {
  if (g.n_obj < 1 || g.n_obj > 65535 || g.n_rows < 1 || g.n_rays < 1 || g.n_samples < 1 || g.n_pix_draw < 1 ||
      g.n_rays % g.n_pix_draw != 0 || g.kf_stride < 1 || g.kf_draw_stride < g.n_rays / g.n_pix_draw)
    return VMB_E_ARG;
  if (!g.kf_draw || !g.kf_frame || !g.ray_rows || (long long)g.n_obj * g.n_rays > g.max_ray_rows) return VMB_E_ARG;
  return VMB_OK;
}

// Check group g, a vmb_track_group or vmb_ba_group (their leading fields share names), and fill the step's arguments
// from it: the sample slice, the network, `pose` (the pose or the pose table), the loss weights and status of `a`.
// Returns the group's tile count, or the VMB_E_* code of the failed check.
template <class G, class Args>
static int pose_group_params(vmb_handle* h, const G& g, const double* pose, const Args* a, const char* who, int path,
                             const void* image, TrackParams& tp) {
  constexpr bool BA = std::is_same_v<G, vmb_ba_group>;
  const std::string w(who);
  if (g.hidden != h->H) return fail(h, VMB_E_ARG, w + ": group hidden size differs from the handle's");
  const bool lw = path != POSE_FP32;                  // a tensor-core path: reads the image, S <= 32
  if (path == POSE_LW && !h->lw_ok) return fail(h, VMB_E_UNSUPPORTED, w + ": the layer-wise path needs hidden 64/128/256 and n_freq 6");
  if (path == POSE_FUSED && !h->umma_ok) return fail(h, VMB_E_UNSUPPORTED, w + ": the fused path needs hidden 32 and n_freq 6");
  if constexpr (BA) {
    if (ba_group_ok(g) != VMB_OK) return fail(h, VMB_E_ARG, w + ": bad counts, draw layout, keyframe tables or ray rows");
  } else {
    if (g.n_obj < 1 || g.n_obj > 65535 || g.n_rows < 1 || g.n_rays < 1 || g.n_samples < 1)
      return fail(h, VMB_E_ARG, w + ": bad n_obj / n_rows / n_rays / n_samples");
  }
  bool missing = !g.rows || !g.pcs || !g.z_vals || !g.gt_depth || !g.gt_colour || !g.sem || !g.mask_depth || !g.params ||
                 !g.scale || (lw && !image);
  if constexpr (!BA) missing = missing || !g.partials;
  if (missing) return fail(h, VMB_E_ARG, w + ": missing tensor pointer");
  const int tiles = vmb_track_tiles(g.hidden, g.n_rays, g.n_samples);
  if (lw && (tiles == VMB_E_UNSUPPORTED || g.n_samples > 32)) return fail(h, VMB_E_UNSUPPORTED, w + ": n_samples above 32");
  if (tiles == VMB_E_UNSUPPORTED)
    return fail(h, VMB_E_UNSUPPORTED, w + ": n_samples exceeds the tile size for this hidden size");
  if (tiles < 1) return fail(h, VMB_E_ARG, w + ": bad shape");
  memset(&tp, 0, sizeof(tp));
  if constexpr (!BA) {
    if ((long long)tiles * g.n_obj > g.max_partials) return fail(h, VMB_E_ARG, w + ": partials buffer too small");
    tp.partials = g.partials;
  }
  tp.B = g.n_obj; tp.R = g.n_rays; tp.S = g.n_samples; tp.n_rows = g.n_rows; tp.rows = g.rows;
  tp.pcs = g.pcs; tp.pcs_stride = g.pcs_stride; tp.z = g.z_vals; tp.z_stride = g.z_stride;
  tp.gt_depth = g.gt_depth; tp.gt_depth_stride = g.gt_depth_stride;
  tp.gt_colour = g.gt_colour; tp.gt_colour_stride = g.gt_colour_stride;
  tp.sem = g.sem; tp.sem_stride = g.sem_stride; tp.mask = g.mask_depth; tp.mask_stride = g.mask_stride;
  tp.params = g.params; tp.scale = g.scale; tp.pose = pose;
  tp.cs = a->colour_scaling; tp.os = a->opacity_scaling; tp.status = a->status;
  return tiles;
}

// The step of group `group`: K10 (vmb_track_args) or K11 (vmb_ba_args), on the network path PATH (PosePath).
template <int PATH, class Args>
static int pose_step(vmb_handle* h, const Args* a, int group, const void* image, void* stream, const char* who) {
  constexpr bool BA = std::is_same_v<Args, vmb_ba_args>;
  if (!h) return fail(h, VMB_E_ARG, std::string(who) + ": null handle");
  const int rc0 = pose_args_ok(h, a, who);
  if (rc0 != VMB_OK) return rc0;
  if (group < 0 || group >= a->n_groups) return fail(h, VMB_E_ARG, std::string(who) + ": group index outside [0, n_groups)");
  const auto& g = a->group[group];
  TrackParams tp;
  BaRays x;
  memset(&x, 0, sizeof(x));
  int tiles;
  if constexpr (BA) {
    tiles = pose_group_params(h, g, a->poses, a, who, PATH, image, tp);
    if (tiles < 0) return tiles;
    x.kf_draw = g.kf_draw; x.kf_draw_stride = g.kf_draw_stride; x.kf_frame = g.kf_frame; x.kf_stride = g.kf_stride;
    x.n_pix_draw = g.n_pix_draw; x.n_poses = a->n_poses; x.rows = g.ray_rows;
  } else {
    tiles = pose_group_params(h, g, a->pose, a, who, PATH, image, tp);
    if (tiles < 0) return tiles;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if constexpr (PATH == POSE_FUSED) {
    std::string err;
    const int rc = tf::launch_track_fused<BA>(h->ws_tf, h->L, tp, x, image, fp32_tile(32) / g.n_samples, h->max_obj,
                                              st, err);
    if (rc != VMB_OK) return fail(h, rc, std::string(who) + ": " + err);
    return VMB_OK;
  } else if constexpr (PATH == POSE_LW) {
    const lw::TlwGroup G{tp, x, (const __half*)image, BA ? 1 : fp32_tile(g.hidden) / g.n_samples};
    std::string err;
    const int rc = lw::launch_track_lw<BA>(BA ? h->ws_ba : h->ws_track, h->L, G, st, err);
    if (rc != VMB_OK) return fail(h, rc, std::string(who) + ": " + err);
    return VMB_OK;
  } else {
    switch (h->H) {
      case 32:  return launch_pose<32, fp32_tile(32), BA>(h, tp, x, tiles, st);
      case 64:  return launch_pose<64, fp32_tile(64), BA>(h, tp, x, tiles, st);
      case 128: return launch_pose<128, fp32_tile(128), BA>(h, tp, x, tiles, st);
      case 256: return launch_pose<256, fp32_tile(256), BA>(h, tp, x, tiles, st);
    }
    return fail(h, VMB_E_UNSUPPORTED, std::string(who) + ": unsupported hidden size");
  }
}

// the update's checks and Adam scalars, shared by vmb_track_update and vmb_ba_update
template <class Args>
static int pose_update_scalars(vmb_handle* h, const Args* a, const char* who, PoseUpdateScalars& s) {
  if (!(std::isfinite(a->lr_rot) && a->lr_rot >= 0.0 && std::isfinite(a->lr_trans) && a->lr_trans >= 0.0 &&
        a->beta1 >= 0.0 && a->beta1 < 1.0 && a->beta2 >= 0.0 && a->beta2 < 1.0 && a->eps > 0.0 && std::isfinite(a->eps)))
    return fail(h, VMB_E_ARG, std::string(who) + ": need finite rates >= 0, betas in [0, 1) and eps > 0");
  for (int c = 0; c < 3; ++c) { s.lr[c] = a->lr_rot; s.lr[3 + c] = a->lr_trans; }
  s.b1 = a->beta1; s.b2 = a->beta2; s.eps = a->eps;
  s.bc1 = 1.0 - std::pow(a->beta1, (double)a->iter);
  s.bc2 = 1.0 - std::pow(a->beta2, (double)a->iter);
  s.cs = a->colour_scaling; s.os = a->opacity_scaling;
  return VMB_OK;
}

extern "C" {

int vmb_track_tiles(int hidden, int n_rays, int n_samples) {
  if (!(hidden == 32 || hidden == 64 || hidden == 128 || hidden == 256) || n_rays < 1 || n_samples < 1) return VMB_E_ARG;
  const int TP = fp32_tile(hidden);
  if (n_samples > TP || n_samples > 32) return VMB_E_UNSUPPORTED;
  const int nr = TP / n_samples;
  return (n_rays + nr - 1) / nr;
}

int vmb_track_step(vmb_handle* h, const vmb_track_args* a, int group, void* stream) {
  return pose_step<POSE_FP32>(h, a, group, nullptr, stream, "vmb_track_step");
}

int vmb_ba_step(vmb_handle* h, const vmb_ba_args* a, int group, void* stream) {
  return pose_step<POSE_FP32>(h, a, group, nullptr, stream, "vmb_ba_step");
}

int vmb_track_step_lw(vmb_handle* h, const vmb_track_args* a, int group, const void* image, void* stream) {
  return pose_step<POSE_LW>(h, a, group, image, stream, "vmb_track_step_lw");
}

int vmb_ba_step_lw(vmb_handle* h, const vmb_ba_args* a, int group, const void* image, void* stream) {
  return pose_step<POSE_LW>(h, a, group, image, stream, "vmb_ba_step_lw");
}

int vmb_track_step_fused(vmb_handle* h, const vmb_track_args* a, int group, const void* image, void* stream) {
  return pose_step<POSE_FUSED>(h, a, group, image, stream, "vmb_track_step_fused");
}

int vmb_ba_step_fused(vmb_handle* h, const vmb_ba_args* a, int group, const void* image, void* stream) {
  return pose_step<POSE_FUSED>(h, a, group, image, stream, "vmb_ba_step_fused");
}

int vmb_reloc_score(vmb_handle* h, const vmb_track_args* a, int group, int n_hyp, const double* hyps, double* scores,
                    double* terms, const void* image, void* stream) {
  const char* who = "vmb_reloc_score";
  if (!h) return fail(h, VMB_E_ARG, std::string(who) + ": null handle");
  if (!a || a->n_groups < 1 || a->n_groups > VMB_TRACK_MAX_GROUPS || group < 0 || group >= a->n_groups)
    return fail(h, VMB_E_ARG, std::string(who) + ": null arguments or group index outside [0, n_groups)");
  if (n_hyp < 1 || n_hyp > VMB_RELOC_MAX_HYP || !hyps || !scores)
    return fail(h, VMB_E_ARG, std::string(who) + ": need 1 <= n_hyp <= VMB_RELOC_MAX_HYP, hyps and scores");
  const auto& g = a->group[group];
  TrackParams tp;
  const int tiles = pose_group_params(h, g, hyps, a, who, POSE_FUSED, image, tp);
  if (tiles < 0) return tiles;
  std::string err;
  const int rc = rl::launch_reloc_fused(h->ws_reloc, h->L, tp, image, hyps, n_hyp, scores, terms,
                                        fp32_tile(32) / g.n_samples, h->n_sm, (cudaStream_t)stream, err);
  if (rc != VMB_OK) return fail(h, rc, std::string(who) + ": " + err);
  return VMB_OK;
}

int vmb_reloc_select(vmb_handle* h, int n, const double* scores, const double* hyps, int k, int* idx, double* poses,
                     void* stream) {
  if (n < 1 || n > VMB_RELOC_MAX_HYP || k < 1 || k > VMB_RELOC_MAX_K || k > n || !scores || !idx || (poses && !hyps))
    return fail(h, VMB_E_ARG, "vmb_reloc_select: need 1 <= k <= min(n, VMB_RELOC_MAX_K), n <= VMB_RELOC_MAX_HYP, "
                              "scores, idx, and hyps when poses are asked for");
  rl::k_reloc_select<<<(unsigned)((n + 255) / 256), 256, (size_t)n * sizeof(double), (cudaStream_t)stream>>>(
      n, scores, hyps, k, idx, poses);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_track_update(vmb_handle* h, const vmb_track_args* a, void* stream) {
  if (!h) return fail(h, VMB_E_ARG, "vmb_track_update: null handle");
  const int rc0 = pose_args_ok(h, a, "vmb_track_update");
  if (rc0 != VMB_OK) return rc0;
  if (!a->adam) return fail(h, VMB_E_ARG, "vmb_track_update: adam state is NULL");
  TrackUpdateParams u;
  memset(&u, 0, sizeof(u));
  const int rc1 = pose_update_scalars(h, a, "vmb_track_update", u.s);
  if (rc1 != VMB_OK) return rc1;
  u.n_groups = a->n_groups;
  for (int i = 0; i < a->n_groups; ++i) {
    const vmb_track_group& g = a->group[i];
    const int tiles = vmb_track_tiles(g.hidden, g.n_rays, g.n_samples);
    if (tiles < 1 || g.n_obj < 1 || !g.partials || (long long)tiles * g.n_obj > g.max_partials)
      return fail(h, tiles == VMB_E_UNSUPPORTED ? VMB_E_UNSUPPORTED : VMB_E_ARG, "vmb_track_update: bad group");
    u.g[i].partials = g.partials; u.g[i].n_obj = g.n_obj; u.g[i].tiles = tiles; u.g[i].loss_terms = g.loss_terms;
  }
  u.iter = a->iter; u.pose = a->pose; u.adam = a->adam;
  u.loss = a->loss; u.pose_hist = a->pose_hist; u.grad_hist = a->grad_hist; u.status = a->status;
  k_track_update<<<1, 256, 0, (cudaStream_t)stream>>>(u);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

int vmb_ba_update(vmb_handle* h, const vmb_ba_args* a, void* stream) {
  if (!h) return fail(h, VMB_E_ARG, "vmb_ba_update: null handle");
  const int rc0 = pose_args_ok(h, a, "vmb_ba_update");
  if (rc0 != VMB_OK) return rc0;
  if (!a->adam || !a->window || !a->scratch) return fail(h, VMB_E_ARG, "vmb_ba_update: adam, window or scratch is NULL");
  if (a->n_win < 1 || a->n_win > VMB_BA_MAX_WIN) return fail(h, VMB_E_ARG, "vmb_ba_update: n_win outside [1, 1024]");
  BaUpdateParams u;
  memset(&u, 0, sizeof(u));
  const int rc1 = pose_update_scalars(h, a, "vmb_ba_update", u.s);
  if (rc1 != VMB_OK) return rc1;
  u.n_groups = a->n_groups;
  long long n_seg = 0;
  for (int i = 0; i < a->n_groups; ++i) {
    const vmb_ba_group& g = a->group[i];
    if (ba_group_ok(g) != VMB_OK) return fail(h, VMB_E_ARG, "vmb_ba_update: bad group");
    u.g[i].rows = g.ray_rows; u.g[i].n_obj = g.n_obj; u.g[i].n_rays = g.n_rays; u.g[i].n_pix_draw = g.n_pix_draw;
    u.g[i].kf_draw = g.kf_draw; u.g[i].kf_draw_stride = g.kf_draw_stride;
    u.g[i].kf_frame = g.kf_frame; u.g[i].kf_stride = g.kf_stride;
    n_seg += (long long)g.n_obj * (g.n_rays / g.n_pix_draw);
  }
  if (8 * n_seg + 6LL * a->n_win > a->scratch_len) return fail(h, VMB_E_ARG, "vmb_ba_update: scratch too small");
  for (int t = 0; t < 2; ++t) {
    const vmb_ba_target& T = a->target[t];
    if (T.t_wc && (!T.frame_of || T.n < 0)) return fail(h, VMB_E_ARG, "vmb_ba_update: target without frame_of");
    u.tgt[t].frame_of = T.frame_of; u.tgt[t].t_wc = T.t_wc; u.tgt[t].n = T.t_wc ? T.n : 0;
  }
  u.iter = a->iter; u.n_iter = a->n_iter; u.n_poses = a->n_poses; u.n_win = a->n_win; u.hold = a->hold;
  u.win = a->window; u.pose = a->poses; u.adam = a->adam; u.scratch = a->scratch;
  u.loss = a->loss; u.pose_hist = a->pose_hist; u.grad_hist = a->grad_hist; u.status = a->status;
  k_ba_update<<<1, 256, 0, (cudaStream_t)stream>>>(u);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

// the pose group of a joint step: it must describe the step's objects, rays and samples (both joint entry points)
static int joint_group(vmb_handle* h, const vmb_step_args* s, const vmb_ba_args* a, int group, const char* who, BaRays& x) {
  const int rc1 = pose_args_ok(h, a, who);
  if (rc1 != VMB_OK) return rc1;
  if (group < 0 || group >= a->n_groups) return fail(h, VMB_E_ARG, std::string(who) + ": group index outside [0, n_groups)");
  const vmb_ba_group& g = a->group[group];
  if (g.hidden != h->H || ba_group_ok(g) != VMB_OK || g.n_obj != s->n_obj || g.n_rays != s->n_rays ||
      g.n_samples != s->n_samples)
    return fail(h, VMB_E_ARG, std::string(who) + ": the pose group must describe the step's objects, rays and samples "
                              "(draw layout, keyframe tables, ray rows)");
  memset(&x, 0, sizeof(x));
  x.kf_draw = g.kf_draw; x.kf_draw_stride = g.kf_draw_stride; x.kf_frame = g.kf_frame; x.kf_stride = g.kf_stride;
  x.n_pix_draw = g.n_pix_draw; x.n_poses = a->n_poses; x.rows = g.ray_rows;
  return VMB_OK;
}

int vmb_joint_step_lw(vmb_handle* h, const vmb_step_args* s, const vmb_ba_args* a, int group, float* pcs_world_out,
                      void* stream) {
  const char* who = "vmb_joint_step_lw";
  StepParams sp;
  const int rc0 = step_params(h, s, sp, who);
  if (rc0 != VMB_OK) return rc0;
  if (!h->lw_ok)
    return fail(h, VMB_E_UNSUPPORTED, "vmb_joint_step_lw: layer-wise path only (hidden 64/128/256, n_freq 6); hidden 32 has "
                                      "no pose gradient from its mapping step");
  if (!s->image || !s->grads || !s->backward || s->fuse_adam || (s->impl != VMB_IMPL_AUTO && s->impl != VMB_IMPL_LAYERWISE))
    return fail(h, VMB_E_ARG, "vmb_joint_step_lw: needs an image, grads, backward = 1, fuse_adam = 0 and the layer-wise impl");
  BaRays x;
  const int rc1 = joint_group(h, s, a, group, who, x);
  if (rc1 != VMB_OK) return rc1;
  cudaStream_t st = (cudaStream_t)stream;
  const int rcc = step_counts(h, s, sp, st);
  if (rcc != VMB_OK) return rcc;
  std::string err;
  const int rc = lw::launch_joint_lw(h->ws, h->ws_joint, h->L, sp, x, a->poses, a->status, s->image, pcs_world_out, st, err);
  if (rc != VMB_OK) return fail(h, rc, std::string(who) + ": " + err);
  if (s->loss_sum) { k_loss_sum<<<1, 32, 0, st>>>(s->loss_terms, s->n_obj, s->loss_sum); CUDA_TRY(h, cudaGetLastError()); }
  return VMB_OK;
}

int vmb_joint_step_fused(vmb_handle* h, const vmb_step_args* s, const vmb_ba_args* a, int group, float* pcs_world_out,
                         void* stream) {
  const char* who = "vmb_joint_step_fused";
  StepParams sp;
  const int rc0 = step_params(h, s, sp, who);
  if (rc0 != VMB_OK) return rc0;
  if (!h->umma_ok)
    return fail(h, VMB_E_UNSUPPORTED, "vmb_joint_step_fused: the fused hidden-32 step only (hidden 32, n_freq 6); hidden "
                                      "64/128/256 take vmb_joint_step_lw");
  if (!s->image || !s->backward || (s->impl != VMB_IMPL_AUTO && s->impl != VMB_IMPL_UMMA))
    return fail(h, VMB_E_ARG, "vmb_joint_step_fused: needs an image, backward = 1 and the fused (umma) impl");
  BaRays x;
  const int rc1 = joint_group(h, s, a, group, who, x);
  if (rc1 != VMB_OK) return rc1;
  cudaStream_t st = (cudaStream_t)stream;
  const long long np = (long long)s->n_rays * s->n_samples;
  const size_t Pp = (size_t)lw::pad_points(np * s->n_obj);
  const bool capturing = stream_capturing(st);
  CUDA_TRY(h, h->ws_joint.pw.grow(Pp * 3 * sizeof(float), capturing));
  CUDA_TRY(h, h->ws_joint.jdt.grow(Pp * 6 * sizeof(float), capturing));
  lw::TlwObj o;
  memset(&o, 0, sizeof(o));
  o.R = s->n_rays; o.S = s->n_samples; o.n_rows = s->n_obj; o.pcs = s->pcs; o.pose = a->poses; o.status = a->status;
  o.n_pix_draw = x.n_pix_draw; o.n_poses = x.n_poses; o.kf_stride = x.kf_stride; o.kf_draw = x.kf_draw; o.kf_frame = x.kf_frame;
  // world points of all B objects, then the fused step on them (pcs_stride: one dense [R][S][3] block per object)
  CUDA_TRY(h, launch_k(lw::k_joint_world, dim3((unsigned)((np + 255) / 256), (unsigned)s->n_obj), dim3(256), 0, st, o,
                       (long long)s->pcs_stride, (long long)x.kf_draw_stride, s->scale, h->ws_joint.pw, pcs_world_out,
                       (int*)nullptr));
  sp.pcs = h->ws_joint.pw; sp.pcs_stride = np * 3;
  FusedExtra fx;
  const int rc2 = fused_extra(h, s, st, fx);
  if (rc2 != VMB_OK) return rc2;
  std::string err;
  const int rc = fused_launch_step(h->L, sp, fx, s->image, h->n_sm, st, err, h->ws_joint.jdt);
  if (rc != VMB_OK) return fail(h, rc, std::string(who) + ": " + err);
  CUDA_TRY(h, launch_k(lw::k_joint_rows, dim3((unsigned)((s->n_rays + 127) / 128), (unsigned)s->n_obj), dim3(128), 0, st, o,
                       (long long)s->pcs_stride, (long long)x.kf_draw_stride, s->scale, (const float*)h->ws_joint.jdt, x.rows));
  return VMB_OK;
}


}  // extern "C"
