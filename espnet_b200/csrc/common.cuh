// Shared device helpers for the espnet_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define ESPB_OK 0
#define ESPB_ERR_ARG -1
#define ESPB_ERR_CUDA -2
#define ESPB_ERR_TMA -3

#define ESPB_CHECK_LAUNCH()                                         \
  do {                                                              \
    cudaError_t e__ = cudaGetLastError();                           \
    if (e__ != cudaSuccess) { espb_set_error(cudaGetErrorString(e__)); return ESPB_ERR_CUDA; } \
  } while (0)

void espb_set_error(const char* msg);

namespace espb {

constexpr int ACT_NONE = 0, ACT_RELU = 1, ACT_SWISH = 2;

// Programmatic dependent launch for the launch-latency-bound decode step (one beam-search step is ~80 small dependent kernels).
// A kernel launched through launch_pdl may become resident while its stream predecessor still runs; it must execute pdl_wait()
// before its first global-memory access (setup that touches only shared memory / barriers may precede it).  pdl_trigger()
// lets the next kernel in the stream do the same.  Every kernel of the chain waits before it completes, so completion order --
// and with it every read-after-write / write-after-read dependency of plain stream order -- is preserved transitively.
// ESPB_PDL=0 launches with full stream serialisation; griddepcontrol.* are no-ops then.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// 3xTF32 operand split: hi keeps the top 19 bits (sign, 8 exp, 10 mantissa) of the fp32 value,
// lo = x - hi is exactly representable in fp32; both planes are stored as fp32 words whose low
// 13 bits are zero, so the tf32 wgmma consumes them without rounding ambiguity.
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
__device__ __forceinline__ float tf32_lo(float x, float hi) { return __uint_as_float(__float_as_uint(x - hi) & 0xFFFFE000u); }

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  if (act == ACT_SWISH) return v / (1.f + __expf(-v));
  return v;
}
// accurate variants (expf, not __expf) are used where parity with the fp32 reference matters
__device__ __forceinline__ float swish_acc(float v) { return v / (1.f + expf(-v)); }
__device__ __forceinline__ float apply_act_acc(float v, int act) {
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  if (act == ACT_SWISH) return swish_acc(v);
  return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum / max for blockDim.x <= 1024 (multiple of 32). `red` needs 33 floats of smem.
__device__ __forceinline__ float block_sum(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (w == 0) { r = warp_sum(r); if (lane == 0) red[32] = r; }
  __syncthreads();
  return red[32];
}
__device__ __forceinline__ float block_max(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : -INFINITY;
  if (w == 0) { r = warp_max(r); if (lane == 0) red[32] = r; }
  __syncthreads();
  return red[32];
}

// log(exp(a)+exp(b)) as torch.logsumexp computes it for two finite operands.
__device__ __forceinline__ float logaddexp(float a, float b) {
  float m = fmaxf(a, b);
  return m + logf(expf(a - m) + expf(b - m));
}

}  // namespace espb
