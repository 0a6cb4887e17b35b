// Shared definitions for the vmap_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define VMB_NDIRS 21
#define VMB_E1 87            // 3 + 21*(3+1): width of the first embedding slice (trainer.py:16)
#define VMB_MAX_FREQ 8
#define VMB_PI_F 3.14159274101257324f   // float32(np.pi): embedding.py:88 multiplies in fp32

// Offsets (in floats) of one object's tensors inside a param-block row; order =
// OccupancyMap.named_parameters() (model.py:17-52) then UniDirsEmbed.B_layer.weight.
struct VmbLayout {
  int H, nfreq, E, e2;
  int o_Win, o_bin, o_Wm1, o_bm1, o_Wcat, o_bcat, o_Wm2, o_bm2, o_Wa, o_ba, o_Wcl, o_bcl, o_Woc, o_boc, o_B;
  int P, stride;
};

__host__ __device__ inline VmbLayout vmb_make_layout(int H, int nfreq) {
  VmbLayout L;
  L.H = H; L.nfreq = nfreq;
  L.E = 3 + VMB_NDIRS * nfreq;
  L.e2 = L.E - VMB_E1;
  int o = 0;
  L.o_Win = o;  o += H * VMB_E1;
  L.o_bin = o;  o += H;
  L.o_Wm1 = o;  o += H * H;
  L.o_bm1 = o;  o += H;
  L.o_Wcat = o; o += H * (H + VMB_E1);
  L.o_bcat = o; o += H;
  L.o_Wm2 = o;  o += H * H;
  L.o_bm2 = o;  o += H;
  L.o_Wa = o;   o += H;
  L.o_ba = o;   o += 1;
  L.o_Wcl = o;  o += H * (H + L.e2);
  L.o_bcl = o;  o += H;
  L.o_Woc = o;  o += 3 * H;
  L.o_boc = o;  o += 3;
  L.o_B = o;    o += VMB_NDIRS * 3;
  L.P = o;
  L.stride = (o + 31) / 32 * 32;
  return L;
}

__device__ __forceinline__ float vmb_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float vmb_sign(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
