// C ABI of libvmap_b200.so (see include/vmap_b200.h).  Host-side launch logic only.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
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

struct vmb_handle {
  int device, max_obj, H, nfreq;
  int n_sm;
  VmbLayout L;
  int* d_counts;          // [max_obj][4]
  int* d_img_index;       // [P] param index -> half index inside the fp16 image (or -1)
  unsigned int* d_ticket; // last-block ticket of the fused AdamW (device step counter mode)
  unsigned int* d_smax;   // [max_obj] sampler: per-object max sampled depth (order-preserving key)
  float* d_partials;      // fused step: [(max_obj + n_sm)][stride] per-(CTA, object) gradient partials (allocated on first use)
  unsigned int* d_objdone;// fused step: [max_obj] finished-segment counters (self-resetting)
  float2* d_bc;           // AdamW bias corrections per step number for (bc_b1, bc_b2), built on the host in double precision
  double bc_b1, bc_b2;
  int img_halves;
  bool umma_ok;           // hidden 32: fused wgmma kernel + its pre-arranged fp16 image
  bool lw_ok;             // hidden 64/128/256: layer-wise wgmma GEMM path + row-major fp16 image
  lw::Workspace ws;       // training-step activations (may be baked into a captured graph)
  lw::Workspace ws_fwd;   // forward-only queries (vmb_forward): separate, so eval_points never moves the step's buffers
  mesh::Workspace ws_mesh;// marching cubes / unprojection scratch (grow-only)
  eval3d::Workspace ws_eval;// box crop / surface sampling / nearest-neighbour scratch (grow-only)
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

template <int H, int TP>
static int launch_fp32(vmb_handle* h, const StepParams& sp, long long n_tiles_x, cudaStream_t st) {
  const size_t smem = step_fp32_smem<H, TP>(h->L);
  static bool attr_set[64] = {};          // per device (one process may drive several GPUs)
  if (!attr_set[h->device & 63]) {
    CUDA_TRY(h, cudaFuncSetAttribute(k_step_fp32<H, TP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[h->device & 63] = true;
  }
  dim3 grid((unsigned)n_tiles_x, (unsigned)sp.B);
  k_step_fp32<H, TP><<<grid, 128, smem, st>>>(sp, h->L);
  CUDA_TRY(h, cudaGetLastError());
  return VMB_OK;
}

static int dispatch_fp32(vmb_handle* h, const StepParams& sp, cudaStream_t st) {
  const int TP = (h->H == 32) ? 128 : (h->H == 256 ? 32 : 64);
  if (sp.S > TP) return fail(h, VMB_E_UNSUPPORTED, "fp32 step kernel: n_samples exceeds the tile size for this hidden size");
  const int nr = TP / sp.S;
  const long long tiles = ((long long)sp.R + nr - 1) / nr;
  if (tiles > 0x7fffffffLL || sp.B > 65535) return fail(h, VMB_E_ARG, "grid too large");
  switch (h->H) {
    case 32:  return launch_fp32<32, 128>(h, sp, tiles, st);
    case 64:  return launch_fp32<64, 64>(h, sp, tiles, st);
    case 128: return launch_fp32<128, 64>(h, sp, tiles, st);
    case 256: return launch_fp32<256, 32>(h, sp, tiles, st);
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
  h->n_sm = 132;
  cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device);
  h->L = vmb_make_layout(hidden, n_freq);
  h->d_counts = nullptr; h->d_img_index = nullptr; h->d_ticket = nullptr; h->d_smax = nullptr; h->d_partials = nullptr; h->d_objdone = nullptr; h->d_bc = nullptr; h->bc_b1 = h->bc_b2 = -1.0; h->img_halves = 0; h->umma_ok = false; h->lw_ok = false;
  cudaError_t e = cudaMalloc(&h->d_counts, sizeof(int) * 4 * max_obj);
  if (e == cudaSuccess) e = cudaMalloc(&h->d_ticket, sizeof(unsigned int));
  if (e == cudaSuccess) e = cudaMemset(h->d_ticket, 0, sizeof(unsigned int));
  if (e == cudaSuccess) e = cudaMalloc(&h->d_smax, sizeof(unsigned int) * (size_t)max_obj);
  if (e != cudaSuccess) { delete h; return fail(nullptr, VMB_E_NOMEM, cudaGetErrorString(e)); }
  if (hidden == 32 && n_freq == 6) {
    std::vector<int> idx(h->L.P);
    umma_fill_image_index(h->L, idx.data());
    h->img_halves = umma_image_bytes() / 2;
    e = cudaMalloc(&h->d_img_index, sizeof(int) * h->L.P);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_img_index, idx.data(), sizeof(int) * h->L.P, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(h->d_counts); delete h; return fail(nullptr, VMB_E_CUDA, cudaGetErrorString(e)); }
    h->umma_ok = true;
  } else if ((hidden == 64 || hidden == 128 || hidden == 256) && n_freq == 6) {
    std::vector<int> idx(h->L.P);
    lw::fill_image_index(h->L, idx.data());
    h->img_halves = (int)lw::img_halves(hidden);
    e = cudaMalloc(&h->d_img_index, sizeof(int) * h->L.P);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_img_index, idx.data(), sizeof(int) * h->L.P, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(h->d_counts); delete h; return fail(nullptr, VMB_E_CUDA, cudaGetErrorString(e)); }
    h->lw_ok = true;
  }
  *out = h;
  return VMB_OK;
}

void vmb_destroy(vmb_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->d_counts) cudaFree(h->d_counts);
  if (h->d_img_index) cudaFree(h->d_img_index);
  if (h->d_ticket) cudaFree(h->d_ticket);
  if (h->d_smax) cudaFree(h->d_smax);
  if (h->d_partials) cudaFree(h->d_partials);
  if (h->d_objdone) cudaFree(h->d_objdone);
  if (h->d_bc) cudaFree(h->d_bc);
  h->ws.release(); h->ws.destroy_streams();
  h->ws_fwd.release(); h->ws_fwd.destroy_streams();
  h->ws_mesh.release();
  h->ws_eval.release();
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

// scratch of the fused step kernel (gradient partial rows + per-object arrival counters): allocated on first use,
// never while a stream capture is in progress (a captured graph bakes the pointers in)
static int fused_scratch(vmb_handle* h, cudaStream_t st) {
  if (h->d_partials) return VMB_OK;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  if (cs != cudaStreamCaptureStatusNone)
    return fail(h, VMB_E_CUDA, "vmb_step: first fused step of a handle must run outside stream capture (scratch allocation)");
  const size_t rows = (size_t)fused_rows_needed(h->max_obj, h->n_sm);
  cudaError_t e = cudaMalloc(&h->d_partials, rows * h->L.stride * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->d_objdone, sizeof(unsigned int) * (2 * (size_t)h->max_obj + 8));
  if (e == cudaSuccess) e = cudaMemset(h->d_objdone, 0, sizeof(unsigned int) * (2 * (size_t)h->max_obj + 8));
  if (e != cudaSuccess) return fail(h, VMB_E_NOMEM, cudaGetErrorString(e));
  return VMB_OK;
}

// Device table of AdamW's bias corrections (1 - b1^t, sqrt(1 - b2^t)) for t < BC_N, computed in double precision like
// torch.optim.adamw does; the kernels index it with the per-object device step number.  Rebuilt when the betas change
// (never during stream capture: a captured graph would keep using the pointer, whose CONTENT is what changes).
constexpr int BC_N = 20480;
static int ensure_bc_table(vmb_handle* h, double b1, double b2, cudaStream_t st) {
  if (h->d_bc && h->bc_b1 == b1 && h->bc_b2 == b2) return VMB_OK;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  if (cs != cudaStreamCaptureStatusNone)
    return fail(h, VMB_E_CUDA, "AdamW bias-correction table must be built outside stream capture (run one step eagerly first)");
  if (!h->d_bc) CUDA_TRY(h, cudaMalloc(&h->d_bc, sizeof(float2) * BC_N));
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

int vmb_step(vmb_handle* h, const vmb_step_args* a, void* stream) {
  if (!h || !a) return fail(h, VMB_E_ARG, "vmb_step: null argument");
  if (a->n_obj <= 0 || a->n_obj > h->max_obj || a->n_rays <= 0 || a->n_samples <= 0 || a->n_samples > 32)
    return fail(h, VMB_E_ARG, "vmb_step: bad n_obj / n_rays / n_samples (1 <= S <= 32)");
  if (!a->pcs || !a->z_vals || !a->gt_depth || !a->gt_colour || !a->sem || !a->mask_depth || !a->params ||
      !a->scale || !a->loss_terms || (a->backward && !a->grads && !a->fuse_adam))
    return fail(h, VMB_E_ARG, "vmb_step: missing tensor pointer");
  if (a->fuse_adam && (!a->backward || !a->exp_avg || !a->exp_avg_sq || (a->step < 1 && !a->step_counter)))
    return fail(h, VMB_E_ARG, "vmb_step: fuse_adam needs backward = 1, exp_avg / exp_avg_sq and a step number");
  cudaStream_t st = (cudaStream_t)stream;
  int impl = a->impl;
  const bool umma_possible = h->umma_ok && a->image != nullptr;
  const bool lw_possible = h->lw_ok && a->image != nullptr;
  if (impl == VMB_IMPL_AUTO) impl = umma_possible ? VMB_IMPL_UMMA : (lw_possible ? VMB_IMPL_LAYERWISE : VMB_IMPL_FP32);
  StepParams sp;
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
  AdamScalars q;
  memset(&q, 0, sizeof(q));
  if (a->fuse_adam) q = adam_scalars(a->lr, a->beta1, a->beta2, a->weight_decay, a->step);
  struct EvGuard {      // records the optional K1 timing events around whichever kernel runs
    cudaEvent_t stop; cudaStream_t st;
    ~EvGuard() { if (stop) cudaEventRecord(stop, st); }
  };

  // ---- hidden 32: ONE launch (counts + step + ordered gradient reduction (+ AdamW)) ----------------------------
  if (impl == VMB_IMPL_UMMA) {
    if (!umma_possible) return fail(h, VMB_E_UNSUPPORTED, "vmb_step: tensor-core path needs hidden=32, n_freq=6 and an image");
    const int rc0 = fused_scratch(h, st);
    if (rc0 != VMB_OK) return rc0;
    FusedExtra fx;
    memset(&fx, 0, sizeof(fx));
    fx.partials = h->d_partials; fx.obj_done = h->d_objdone; fx.counts_in = a->counts; fx.counts_pub = h->d_counts;
    fx.fuse_adam = a->fuse_adam ? 1 : 0;
    if (a->fuse_adam) {
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
    EvGuard evg{(cudaEvent_t)a->k1_stop_event, st};
    if (a->k1_start_event) cudaEventRecord((cudaEvent_t)a->k1_start_event, st);
    std::string err;
    fx.loss_sum = a->loss_sum;
    bool coop = false;
    const int rc = fused_launch_step(h->L, sp, fx, a->image, h->n_sm, st, err, &coop);
    if (rc != VMB_OK) return fail(h, rc, err);
    if (a->loss_sum && !coop) { k_loss_sum<<<1, 32, 0, st>>>(a->loss_terms, a->n_obj, a->loss_sum); CUDA_TRY(h, cudaGetLastError()); }
    return VMB_OK;
  }

  // ---- other paths: K0 (mask counts) -> K1 -> [K2] ---------------------------------------------------------------
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
  if (a->backward && !a->grads) return fail(h, VMB_E_ARG, "vmb_step: this path needs the grads block");
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
    if (rc) return fail(h, rc == -4 ? VMB_E_UNSUPPORTED : VMB_E_CUDA, err);
    return VMB_OK;
  }
  if (a->image && h->lw_ok) {
    std::string err;
    const int rc = lw::launch_forward(h->ws_fwd, h->L, sp, a->image, (cudaStream_t)stream, err);
    if (rc) return fail(h, rc == -4 ? VMB_E_UNSUPPORTED : VMB_E_CUDA, err);
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
  static bool attr_set[64] = {};
  if (!attr_set[h->device & 63]) {
    CUDA_TRY(h, cudaFuncSetAttribute(k_sample_points<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 256 * 32 * 16));
    CUDA_TRY(h, cudaFuncSetAttribute(k_sample_points<1, 9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 256 * 32 * 16));
    CUDA_TRY(h, cudaFuncSetAttribute(k_sample_points<5, 9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 256 * 32 * 16));
    attr_set[h->device & 63] = true;
  }
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
  const size_t n1 = (size_t)q.n + 1;
  CUDA_TRY(h, mesh::Workspace::grow((void**)&w.mc_bytes, &w.mc_cap, 2 * n1 * sizeof(int) + 2 * (size_t)q.n));
  q.pt_scan = reinterpret_cast<int*>(w.mc_bytes);
  q.cell_scan = q.pt_scan + n1;
  q.pt_mask = reinterpret_cast<unsigned char*>(q.cell_scan + n1);
  q.cell_case = q.pt_mask + q.n;
  mesh::k_mc_count<<<mesh::blocks_for((long long)n1), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.scan(q.pt_scan, (long long)n1, st));
  CUDA_TRY(h, w.scan(q.cell_scan, (long long)n1, st));
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
  CUDA_TRY(h, mesh::Workspace::grow((void**)&w.up_scan, &w.up_cap, (size_t)(q.n + 1) * sizeof(int)));
  q.scan = w.up_scan;
  mesh::k_unproj_flag<<<mesh::blocks_for(q.n + 1), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.scan(q.scan, q.n + 1, st));
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
  CUDA_TRY(h, eval3d::Workspace::grow((void**)&w.clip_scan, &w.clip_cap, (size_t)(q.nf + 1) * sizeof(int)));
  q.scan = w.clip_scan;
  eval3d::k_clip_count<<<eval3d::blocks_for(q.nf + 1, 128), 128, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.exclusive_sum(q.scan, q.nf + 1, st));
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
  CUDA_TRY(h, eval3d::Workspace::grow((void**)&w.cum, &w.cum_cap, (size_t)q.nf * sizeof(double) + sizeof(double)));
  q.cum = w.cum;
  q.bad = reinterpret_cast<int*>(w.cum + q.nf);
  CUDA_TRY(h, cudaMemsetAsync(q.bad, 0, sizeof(int), st));
  eval3d::k_face_area<<<eval3d::blocks_for(q.nf, 256), 256, 0, st>>>(q);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, w.inclusive_sum(q.cum, q.nf, st));
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
  CUDA_TRY(h, eval3d::Workspace::grow((void**)&w.nn, &w.nn_cap, need));
  q.keys = reinterpret_cast<unsigned int*>(w.nn);
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
  CUDA_TRY(h, w.exclusive_sum(q.cell_start, q.max_cells + 1, st));
  eval3d::k_nn_scatter<<<eval3d::blocks_for(q.n_ref, 256), 256, 0, st>>>(q);
  eval3d::k_nn_query<<<eval3d::blocks_for(q.n_q, 128), 128, 0, st>>>(q);
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
