// Kernels of the language model's full-sequence forward and its perplexity (espnet2/lm/espnet_model.py:24-70,
// espnet2/bin/lm_calc_perplexity.py): the causal, token-masked softmax of the materialised attention path (d_k != 64; d_k = 64 runs the
// fused kernel of attention.cu) and the fused negative log-likelihood of the output logits.
#include <math.h>

#include "common.cuh"

namespace {

__device__ __forceinline__ void store_split(float* p, long long plane, float v) {
  const float hi = espb::tf32_hi(v);
  p[0] = hi;
  p[plane] = espb::tf32_lo(v, hi);
}

// One warp per row (b, h, i): probs = softmax(scores / sqrt_dk) over the keys j <= i, j < lens[b] with tok[b][j] != 0, 0 elsewhere (also
// on rows without a valid key) -- TransformerLM._target_mask (transformer_lm.py:57-60) through MultiHeadedAttention.forward_attention
// (attention.py:121-151).
__global__ void __launch_bounds__(256) causal_softmax_kernel(const float* __restrict__ sc, int B, int H, int T, int Tp, const int* __restrict__ lens,
                                                             const int* __restrict__ tok, float scale_div, float* __restrict__ probs,
                                                             long long probs_plane) {
  const long long rowid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (rowid >= (long long)B * H * T) return;
  const int lane = threadIdx.x & 31;
  const int i = (int)(rowid % T), b = (int)(rowid / ((long long)H * T));
  const int nk = min(lens[b], i + 1);
  const int* tk = tok + (long long)b * T;
  const float* ar = sc + rowid * Tp;
  float* pr = probs + rowid * Tp;
  float mx = -INFINITY;
  for (int j = lane; j < nk; j += 32)
    if (tk[j] != 0) mx = fmaxf(mx, ar[j] / scale_div);
  mx = espb::warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < nk; j += 32)
    if (tk[j] != 0) sum += expf(ar[j] / scale_div - mx);
  sum = espb::warp_sum(sum);
  for (int j = lane; j < Tp; j += 32) {
    float p = 0.f;
    if (j < nk && tk[j] != 0) p = expf(ar[j] / scale_div - mx) / sum;
    store_split(pr + j, probs_plane, p);
  }
}

// (max, sum of exp(x - max)) of two parts of a row
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  if (mn == -INFINITY) return;
  s = s * expf(m - mn) + s2 * expf(m2 - mn);
  m = mn;
}

__device__ __forceinline__ void lse_add(float& m, float& s, float x) {
  if (x > m) {
    s = s * expf(m - x) + 1.f;
    m = x;
  } else {
    s += expf(x - m);
  }
}

// One block per row r: out[r] = logsumexp(x[r][0..V-1]) - x[r][tgt[r]] in fp32 (F.cross_entropy, reduction "none"), read in one pass with a
// running max; 0 where tgt[r] < 0 (padding), NaN where tgt[r] >= V.
template <bool VEC4>
__global__ void __launch_bounds__(256) nll_rows_kernel(const float* __restrict__ x, long long ld, int V, const int* __restrict__ tgt,
                                                       float* __restrict__ out) {
  __shared__ float red_m[8], red_s[8];
  const long long r = blockIdx.x;
  const int t = tgt[r];
  if (t < 0) {
    if (threadIdx.x == 0) out[r] = 0.f;
    return;
  }
  const float* row = x + r * ld;
  float m = -INFINITY, s = 0.f;
  if (VEC4) {
    const float4* row4 = reinterpret_cast<const float4*>(row);
    for (int j = threadIdx.x; j < V / 4; j += blockDim.x) {
      const float4 v = __ldg(row4 + j);
      lse_add(m, s, v.x); lse_add(m, s, v.y); lse_add(m, s, v.z); lse_add(m, s, v.w);
    }
  } else {
    for (int j = threadIdx.x; j < V; j += blockDim.x) lse_add(m, s, __ldg(row + j));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red_m[w] = m; red_s[w] = s; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) lse_merge(m, s, red_m[k], red_s[k]);
    // -(log_softmax(x)[t]) = log(sum) - (x[t] - max), the order ATen's log_softmax rounds in
    out[r] = t < V ? logf(s) - (row[t] - m) : NAN;
  }
}

}  // namespace

extern "C" {

int espb_causal_softmax_f32(const float* scores, int B, int H, int T, int Tp, const int* lens, const int* tok, float sqrt_dk, float* probs,
                            long long probs_plane, cudaStream_t stream) {
  if (B <= 0 || H <= 0 || T <= 0) return ESPB_OK;
  if (Tp < T || !tok) { espb_set_error("causal_softmax: need Tp >= T and token ids"); return ESPB_ERR_ARG; }
  const long long rows = (long long)B * H * T;
  causal_softmax_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(scores, B, H, T, Tp, lens, tok, sqrt_dk, probs, probs_plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_nll_rows_f32(const float* x, long long rows, long long ld, int V, const int* tgt, float* out, cudaStream_t stream) {
  if (rows <= 0) return ESPB_OK;
  if (V <= 0 || ld < V) { espb_set_error("nll_rows: need 0 < V <= ld"); return ESPB_ERR_ARG; }
  if ((ld & 3) == 0 && (V & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0)
    nll_rows_kernel<true><<<(unsigned)rows, 256, 0, stream>>>(x, ld, V, tgt, out);
  else
    nll_rows_kernel<false><<<(unsigned)rows, 256, 0, stream>>>(x, ld, V, tgt, out);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

}  // extern "C"
