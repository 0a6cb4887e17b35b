// K2: fused stacked AdamW over the packed [n_obj][stride] fp32 param block.
// Restates torch.optim.AdamW.step() as the reference drives it (train.py:67,325-326;
// groups added by utils.py:33): decoupled decay on every tensor, default betas/eps,
// one shared step counter (all stacked tensors are always stepped together), followed by
// zero_grad.  Optionally refreshes the fp16 tensor-core weight image consumed by the
// UMMA step kernel, so K1 can stage an object's weights with one bulk copy.
#pragma once
#include "common.cuh"

struct AdamParams {
  long long n;                // B * stride
  int stride, P;              // row pitch, live floats per row
  int B;
  float* p; float* g; float* m; float* v;
  __half* image; const int* img_index; int img_halves;   // per-object image size in halves
  const float* loss_terms; int* status;
  const float* grad_scale;    // optional device scalar multiplied into the gradients as they are read
  const float* loss_sum_src; float* loss_sum;   // optional: block 0 writes sum_b loss_sum_src[b][3] (the step's scalar loss)
  float lr_wd;                // 1 - lr*wd
  float one_m_b1, b2, one_m_b2;
  float step_size;            // lr / (1 - b1^t)
  float bc2_sqrt;             // sqrt(1 - b2^t)
  float eps;
  int zero_grads;
  // optional device-resident per-object step numbers (CUDA-graph replay): t_b = step_counter[b] + 1 is read by
  // every block on entry; the last block to finish increments those of the updated objects and resets the ticket.
  int* step_counter; unsigned int* ticket;
  double lr, b1, b2d;
  float log_b1, log_b2;       // ln(beta1), ln(beta2)
  const float2* bc_table; int bc_n;   // [t] -> (1 - beta1^t, sqrt(1 - beta2^t)), host-built in double precision
};

// render_rays.py:88-90's guard on object b's loss terms (the reference aborts before the update): 1 = one of the three
// terms above 1e5, 2 = any of the four values (terms and weighted total) non-finite or beyond 3e38; 0 when the guard is
// off.  The fused hidden-32 finisher tests only the total for bit 2; a non-finite term always makes the total
// non-finite, so both flag the same objects.
__device__ __forceinline__ int adam_row_guard(const float* loss_terms, int b) {
  if (!loss_terms) return 0;
  int bad = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float l = loss_terms[b * 4 + i];
    if (i != 3 && l > 100000.f) bad |= 1;
    if (!(l == l) || fabsf(l) > 3.0e38f) bad |= 2;
  }
  return bad;
}

// The guard is per object: a row whose loss tripped it keeps its params, moments, image and step number and only has
// its gradients zeroed; the other rows of the launch are updated.
__global__ void __launch_bounds__(256) k_adamw(AdamParams a) {
  __shared__ int s_skip[2];
  __shared__ float s_step_size[2], s_bc2_sqrt[2];
  // issue this thread's loads first: their latency overlaps the bias-correction prologue
  const long long i4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f), g = p, m = p, v = p;
  if (i4 < a.n) {
    p = *reinterpret_cast<const float4*>(a.p + i4);
    g = *reinterpret_cast<const float4*>(a.g + i4);
    m = *reinterpret_cast<const float4*>(a.m + i4);
    v = *reinterpret_cast<const float4*>(a.v + i4);
  }
  // a block covers 1024 consecutive floats = at most two rows (row pitch >= 1024): per-object step numbers
  const int row0 = (int)(((long long)blockIdx.x * blockDim.x * 4) / a.stride);
  if (threadIdx.x < 2) {
    const int rb = row0 + threadIdx.x;
    const int bad = rb < a.B ? adam_row_guard(a.loss_terms, rb) : 0;
    s_skip[threadIdx.x] = bad;
    // the block holding the row's first float reports it, so the status word gets each row's bits exactly once
    if (bad && a.status && (long long)rb * a.stride / ((long long)blockDim.x * 4) == blockIdx.x) atomicOr(a.status, bad);
    if (a.step_counter && rb < a.B) {
      // bias corrections of step t from the host-built table (torch's double scalars, rounded once); beyond the table
      // 1 - beta^t = -expm1(t ln beta), fp32, cancellation-free (<= 3e-7 relative)
      const int t = a.step_counter[rb] + 1;
      if (t < a.bc_n) {
        const float2 bc = a.bc_table[t];
        s_step_size[threadIdx.x] = (float)a.lr / bc.x;
        s_bc2_sqrt[threadIdx.x] = bc.y;
      } else {
        s_step_size[threadIdx.x] = (float)a.lr / (-expm1f((float)t * a.log_b1));
        s_bc2_sqrt[threadIdx.x] = sqrtf(-expm1f((float)t * a.log_b2));
      }
    } else {
      s_step_size[threadIdx.x] = a.step_size; s_bc2_sqrt[threadIdx.x] = a.bc2_sqrt;
    }
  }
  if (a.loss_sum && blockIdx.x == 0 && threadIdx.x >= 32 && threadIdx.x < 64) {
    float s = 0.f;
    for (int b = threadIdx.x - 32; b < a.B; b += 32) s += a.loss_sum_src[b * 4 + 3];
    s = warp_sum(s);
    if (threadIdx.x == 32) *a.loss_sum = s;
  }
  __syncthreads();
  const int b = (int)(i4 / a.stride);
  if (i4 < a.n && s_skip[b - row0]) {
    // no update of this object; its exploded gradients must not leak into the next step's accumulation
    if (a.zero_grads) *reinterpret_cast<float4*>(a.g + i4) = make_float4(0.f, 0.f, 0.f, 0.f);
  } else if (i4 < a.n) {
  if (a.grad_scale) { const float gs = *a.grad_scale; g.x *= gs; g.y *= gs; g.z *= gs; g.w *= gs; }
  const float step_size = s_step_size[b - row0], bc2_sqrt = s_bc2_sqrt[b - row0];
  float* pp = &p.x; float* gg = &g.x; float* mm = &m.x; float* vv = &v.x;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float pj = pp[j] * a.lr_wd;                                  // p.mul_(1 - lr*wd)
    const float mj = mm[j] + (gg[j] - mm[j]) * a.one_m_b1;       // exp_avg.lerp_(g, 1-b1)
    const float vj = vv[j] * a.b2 + (a.one_m_b2 * gg[j]) * gg[j];// exp_avg_sq.mul_(b2).addcmul_(g,g,1-b2)
    const float denom = sqrtf(vj) / bc2_sqrt + a.eps;
    pj = pj - step_size * (mj / denom);                        // p.addcdiv_(m, denom, -step_size)
    pp[j] = pj; mm[j] = mj; vv[j] = vj;
  }
  *reinterpret_cast<float4*>(a.p + i4) = p;
  *reinterpret_cast<float4*>(a.m + i4) = m;
  *reinterpret_cast<float4*>(a.v + i4) = v;
  if (a.zero_grads) *reinterpret_cast<float4*>(a.g + i4) = make_float4(0.f, 0.f, 0.f, 0.f);
  if (a.image) {
    const int e = (int)(i4 - (long long)b * a.stride);
    __half* img = a.image + (size_t)b * a.img_halves;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (e + j < a.P) {
        const int t = a.img_index[e + j];
        if (t >= 0) img[t] = __float2half_rn(pp[j]);
        else if (t <= -2) reinterpret_cast<float*>(img)[-(t + 2)] = pp[j];
      }
    }
  }
  }
  if (a.step_counter) {
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      s_last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last) {           // every block has read its step numbers: the last one to finish publishes t + 1
      for (int i = threadIdx.x; i < a.B; i += blockDim.x)
        if (!adam_row_guard(a.loss_terms, i)) a.step_counter[i] += 1;
      if (threadIdx.x == 0) *a.ticket = 0u;
    }
  }
}

// fp32 master weights -> fp16 image (init / checkpoint load / re-stack)
__global__ void __launch_bounds__(256) k_build_image(int B, int stride, int P, const float* p,
                                                      __half* image, const int* img_index, int img_halves) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * stride) return;
  const int b = (int)(i / stride), e = (int)(i - (long long)b * stride);
  if (e >= P) return;
  const int t = img_index[e];
  if (t >= 0) image[(size_t)b * img_halves + t] = __float2half_rn(p[i]);
  else if (t <= -2) reinterpret_cast<float*>(image + (size_t)b * img_halves)[-(t + 2)] = p[i];
}
