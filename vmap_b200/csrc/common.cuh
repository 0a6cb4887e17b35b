// Shared definitions for the vmap_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <utility>

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

// ---- host: handle scratch and per-device caches ----------------------------------------------------------------------

// Whether work enqueued on `st` is being captured into a CUDA graph.  An entry point asks once and passes the answer to
// every buffer it grows.
static inline bool stream_capturing(cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cs);
  return cs != cudaStreamCaptureStatusNone;
}

// One grow-only device allocation of handle scratch, freed with its owner.  A graph captured on a stream bakes the
// pointer into its kernel arguments and tensor maps, so a buffer that a capture has used is pinned: it never moves
// again, and a call that needs it larger is refused (cudaErrorStreamCaptureUnsupported) instead of leaving the graph a
// freed pointer.  It converts to its pointer so call sites carve and pass it as the raw pointer it replaces.
template <class T>
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  DeviceBuffer(DeviceBuffer&& o) noexcept : p_(o.p_), bytes_(o.bytes_), pinned_(o.pinned_) { o.p_ = nullptr; o.bytes_ = 0; }
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
    std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); std::swap(pinned_, o.pinned_);
    return *this;
  }
  ~DeviceBuffer() { if (p_) cudaFree(p_); }

  // At least `bytes` bytes.  A buffer that fits is kept, and pinned when `capturing`; one that must grow during a
  // capture, or after one, is refused.  Otherwise the old allocation is replaced; on failure the buffer is left empty.
  cudaError_t grow(size_t bytes, bool capturing) {
    if (bytes <= bytes_) { pinned_ |= capturing; return cudaSuccess; }
    if (capturing || pinned_) return cudaErrorStreamCaptureUnsupported;
    if (p_) cudaFree(p_);
    p_ = nullptr; bytes_ = 0;
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) return e;
    p_ = static_cast<T*>(p); bytes_ = bytes;
    return cudaSuccess;
  }
  T* get() const { return p_; }
  operator T*() const { return p_; }
  size_t bytes() const { return bytes_; }

 private:
  T* p_ = nullptr;
  size_t bytes_ = 0;
  bool pinned_ = false;
};

// host: raise kernel K's dynamic shared-memory limit to `bytes` on device `dev`, the first time only
template <auto K>
static cudaError_t smem_limit_once(int dev, int bytes) {
  static bool set[64] = {};      // per device (one process may drive several GPUs)
  if (set[dev & 63]) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) set[dev & 63] = true;
  return e;
}

// multiprocessors of device `dev` (launch sizing), looked up once; 132 (an H100 SXM) when the query fails
static int sm_count(int dev) {
  static int n[64] = {};
  if (!n[dev & 63] && (cudaDeviceGetAttribute(&n[dev & 63], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
                       n[dev & 63] <= 0))
    n[dev & 63] = 132;
  return n[dev & 63];
}
