// CTC head kernels: row-wise log-softmax / argmax over the vocabulary, on-device greedy collapse, and the row softmax that feeds the
// self-conditioning GEMM of intermediate CTC.
// Reference: espnet2/asr/ctc.py:187-215 (softmax, log_softmax, argmax), espnet2/asr/encoder/conformer_encoder.py:394-414 (conditioning),
// espnet2/bin/asr_inference.py:574-575 and espnet2/bin/s2t_inference_ctc.py:630-632 (unique_consecutive + drop blank).
#include "common.cuh"

namespace {

// In-place log-softmax of each row of x [rows][V] (row pitch ld). One block per row.
__global__ void __launch_bounds__(256) log_softmax_rows_kernel(float* __restrict__ x, long long ld, int V) {
  espb::pdl_trigger();
  espb::pdl_wait();
  __shared__ float red[33];
  float* r = x + (long long)blockIdx.x * ld;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < V; i += blockDim.x) mx = fmaxf(mx, r[i]);
  mx = espb::block_max(mx, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x) s += expf(r[i] - mx);
  s = espb::block_sum(s, red);
  const float lse = mx + logf(s);
  for (int i = threadIdx.x; i < V; i += blockDim.x) r[i] = r[i] - lse;
}

// Same result (same per-thread summation order), one global read: thread t keeps x[t + 256 k], k < NV, in registers (V <= 256 NV).
template <int NV>
__global__ void __launch_bounds__(256) log_softmax_rows_reg_kernel(float* __restrict__ x, long long ld, int V) {
  espb::pdl_trigger();
  espb::pdl_wait();
  __shared__ float red[33];
  float* r = x + (long long)blockIdx.x * ld;
  float v[NV];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = threadIdx.x + k * 256;
    v[k] = (i < V) ? r[i] : -INFINITY;
    mx = fmaxf(mx, v[k]);
  }
  mx = espb::block_max(mx, red);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) if (threadIdx.x + k * 256 < V) s += expf(v[k] - mx);
  s = espb::block_sum(s, red);
  const float lse = mx + logf(s);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = threadIdx.x + k * 256;
    if (i < V) r[i] = v[k] - lse;
  }
}

// Softmax of each row of x [rows][V] (row pitch ld) into the tf32 hi / lo planes out, out + out_plane [rows][ldo] (the A operand of the
// 3xTF32 GEMM), columns V..ldo-1 zero. One block per row; the same per-thread summation order as log_softmax_rows_reg_kernel, with
// x[t + 256 k], k < NV, held in registers (V <= 256 NV).
__device__ __forceinline__ void store_split_row(float* __restrict__ o, long long plane, int i, float p) {
  const float hi = espb::tf32_hi(p);
  o[i] = hi;
  o[plane + i] = espb::tf32_lo(p, hi);
}

__device__ __forceinline__ void zero_split_tail(float* __restrict__ o, long long plane, int V, long long ldo) {
  for (long long i = V + threadIdx.x; i < ldo; i += blockDim.x) { o[i] = 0.f; o[plane + i] = 0.f; }
}

template <int NV>
__global__ void __launch_bounds__(256) softmax_rows_split_reg_kernel(const float* __restrict__ x, long long ld, int V, float* __restrict__ out,
                                                                     long long out_plane, long long ldo) {
  espb::pdl_trigger();
  espb::pdl_wait();
  __shared__ float red[33];
  const float* r = x + (long long)blockIdx.x * ld;
  float* o = out + (long long)blockIdx.x * ldo;
  float v[NV];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = threadIdx.x + k * 256;
    v[k] = (i < V) ? r[i] : -INFINITY;
    mx = fmaxf(mx, v[k]);
  }
  mx = espb::block_max(mx, red);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    v[k] = expf(v[k] - mx);
    if (threadIdx.x + k * 256 < V) s += v[k];
  }
  s = espb::block_sum(s, red);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = threadIdx.x + k * 256;
    if (i < V) store_split_row(o, out_plane, i, v[k] / s);
  }
  zero_split_tail(o, out_plane, V, ldo);
}

// Same result for any V: three passes over the row in global memory (max, sum, store), each thread visiting the same columns in the same order.
__global__ void __launch_bounds__(256) softmax_rows_split_kernel(const float* __restrict__ x, long long ld, int V, float* __restrict__ out,
                                                                 long long out_plane, long long ldo) {
  espb::pdl_trigger();
  espb::pdl_wait();
  __shared__ float red[33];
  const float* r = x + (long long)blockIdx.x * ld;
  float* o = out + (long long)blockIdx.x * ldo;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < V; i += 256) mx = fmaxf(mx, r[i]);
  mx = espb::block_max(mx, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += 256) s += expf(r[i] - mx);
  s = espb::block_sum(s, red);
  for (int i = threadIdx.x; i < V; i += 256) store_split_row(o, out_plane, i, expf(r[i] - mx) / s);
  zero_split_tail(o, out_plane, V, ldo);
}

// argmax of each row (first index on ties, as torch.argmax on CPU). One warp per row.
__global__ void __launch_bounds__(256) argmax_rows_kernel(const float* __restrict__ x, long long rows, long long ld, int V, int* __restrict__ out) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* r = x + row * ld;
  float best = -INFINITY; int bi = 0x7fffffff;
  for (int i = lane; i < V; i += 32) {
    float v = r[i];
    if (v > best || (v == best && i < bi)) { best = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) out[row] = bi;
}

// Greedy collapse per utterance: drop repeats then blanks. One warp per utterance, ballot-compacted.
__global__ void ctc_collapse_kernel(const int* __restrict__ am, int Tmax, const int* __restrict__ lens, int blank, int* __restrict__ out_ids,
                                    int* __restrict__ out_len) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int len = lens[b];
  const int* a = am + (long long)b * Tmax;
  int* o = out_ids + (long long)b * Tmax;
  int n = 0;
  for (int t0 = 0; t0 < len; t0 += 32) {
    int t = t0 + lane;
    bool keep = false; int v = 0;
    if (t < len) {
      v = a[t];
      keep = (v != blank) && (t == 0 || a[t - 1] != v);
    }
    unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) o[n + __popc(m & ((1u << lane) - 1))] = v;
    n += __popc(m);
  }
  if (lane == 0) out_len[b] = n;
}

}  // namespace

extern "C" {

int espb_log_softmax_rows_f32(float* x, long long rows, long long ld, int V, cudaStream_t stream) {
  if (rows <= 0) return ESPB_OK;
  if (V <= 256 * 8) espb::launch_pdl(log_softmax_rows_reg_kernel<8>, dim3((unsigned)rows), dim3(256), 0, stream, x, ld, V);
  else if (V <= 256 * 20) espb::launch_pdl(log_softmax_rows_reg_kernel<20>, dim3((unsigned)rows), dim3(256), 0, stream, x, ld, V);
  else if (V <= 256 * 32) espb::launch_pdl(log_softmax_rows_reg_kernel<32>, dim3((unsigned)rows), dim3(256), 0, stream, x, ld, V);
  else espb::launch_pdl(log_softmax_rows_kernel, dim3((unsigned)rows), dim3(256), 0, stream, x, ld, V);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_softmax_rows_split_f32(const float* x, long long rows, long long ld, int V, float* out, long long out_plane, long long ldo,
                                cudaStream_t stream) {
  if (rows < 0 || V <= 0 || ld < V) { espb_set_error("softmax_rows_split: need rows >= 0, V > 0 and ld >= V"); return ESPB_ERR_ARG; }
  if (ldo < V || ldo % 32) { espb_set_error("softmax_rows_split: ldo must be a multiple of 32 and >= V"); return ESPB_ERR_ARG; }
  if (out_plane < rows * ldo) { espb_set_error("softmax_rows_split: out_plane must be >= rows * ldo"); return ESPB_ERR_ARG; }
  if (rows == 0) return ESPB_OK;
  if (!x || !out) { espb_set_error("softmax_rows_split: null pointer"); return ESPB_ERR_ARG; }
  const dim3 grid((unsigned)rows), block(256);
  if (V <= 256 * 8) espb::launch_pdl(softmax_rows_split_reg_kernel<8>, grid, block, 0, stream, x, ld, V, out, out_plane, ldo);
  else if (V <= 256 * 20) espb::launch_pdl(softmax_rows_split_reg_kernel<20>, grid, block, 0, stream, x, ld, V, out, out_plane, ldo);
  else if (V <= 256 * 32) espb::launch_pdl(softmax_rows_split_reg_kernel<32>, grid, block, 0, stream, x, ld, V, out, out_plane, ldo);
  else espb::launch_pdl(softmax_rows_split_kernel, grid, block, 0, stream, x, ld, V, out, out_plane, ldo);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_argmax_rows_f32(const float* x, long long rows, long long ld, int V, int* out, cudaStream_t stream) {
  if (rows <= 0) return ESPB_OK;
  argmax_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(x, rows, ld, V, out);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_ctc_collapse_i32(const int* argmax, int B, int Tmax, const int* lens, int blank, int* out_ids, int* out_len, cudaStream_t stream) {
  ctc_collapse_kernel<<<B, 32, 0, stream>>>(argmax, Tmax, lens, blank, out_ids, out_len);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

}  // extern "C"
