// Warp-primitive kernels of the Conformer encoder: LayerNorm, conv1 of the 2-D subsampling, rel-pos
// attention glue (q+u / q+v, V transpose, rel-shift + masked softmax) and the convolution module's
// GLU + depthwise conv + BatchNorm(eval) + Swish.  All outputs that feed a GEMM are written as
// tf32 hi/lo planes (see gemm.h).
//
// Reference: espnet2/legacy/nets/pytorch_backend/transformer/{layer_norm,subsampling,attention}.py,
// .../conformer/{convolution,encoder_layer}.py (line ranges at each kernel).
#include <stdint.h>
#include <stdlib.h>

#include "common.cuh"

namespace {

using espb::tf32_hi;
using espb::tf32_lo;

__device__ __forceinline__ void store_split(float* p, long long plane, float v) {
  float h = tf32_hi(v);
  p[0] = h;
  p[plane] = tf32_lo(v, h);
}

// ---------------------------------------------------------------- LayerNorm (layer_norm.py:12-42, eps 1e-12)
// One warp per row, D <= 2048 (D % 32 == 0 not required). out_plain and/or out_split may be null.
template <int MAXV>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, long long rows, int D, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, float* __restrict__ out_plain,
                                                        float* __restrict__ out_split, long long split_plane) {
  espb::pdl_trigger();
  espb::pdl_wait();
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * D;
  float v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = lane + i * 32;
    v[i] = (c < D) ? xr[c] : 0.f;
    s += v[i];
  }
  const float mean = espb::warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = lane + i * 32;
    float d = (c < D) ? v[i] - mean : 0.f;
    q += d * d;
  }
  const float rstd = 1.0f / sqrtf(espb::warp_sum(q) / (float)D + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int c = lane + i * 32;
    if (c < D) {
      float y = (v[i] - mean) * rstd * gamma[c] + beta[c];
      if (out_plain) out_plain[row * D + c] = y;
      if (out_split) store_split(out_split + row * D + c, split_plane, y);
    }
  }
}

// 128-bit variant (D % 4 == 0, 16-byte aligned rows): x, gamma and beta are all requested before the first reduction, so one
// memory round trip covers them; small problems (decode step: a few hundred rows) use 2 rows per block to spread over all SMs.
template <int NV4>
__global__ void __launch_bounds__(256) layernorm_vec_kernel(const float* __restrict__ x, long long rows, int D, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float eps, float* __restrict__ out_plain,
                                                            float* __restrict__ out_split, long long split_plane) {
  espb::pdl_trigger();
  espb::pdl_wait();
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * D;
  float4 v[NV4], g[NV4], b[NV4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    const int c = (lane + i * 32) * 4;
    if (c < D) {
      v[i] = *reinterpret_cast<const float4*>(xr + c);
      g[i] = __ldg(reinterpret_cast<const float4*>(gamma + c));
      b[i] = __ldg(reinterpret_cast<const float4*>(beta + c));
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f); g[i] = v[i]; b[i] = v[i];
    }
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = espb::warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    const int c = (lane + i * 32) * 4;
    if (c < D) {
      const float d0 = v[i].x - mean, d1 = v[i].y - mean, d2 = v[i].z - mean, d3 = v[i].w - mean;
      q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
  }
  const float rstd = 1.0f / sqrtf(espb::warp_sum(q) / (float)D + eps);
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    const int c = (lane + i * 32) * 4;
    if (c < D) {
      float4 y;
      y.x = (v[i].x - mean) * rstd * g[i].x + b[i].x; y.y = (v[i].y - mean) * rstd * g[i].y + b[i].y;
      y.z = (v[i].z - mean) * rstd * g[i].z + b[i].z; y.w = (v[i].w - mean) * rstd * g[i].w + b[i].w;
      if (out_plain) *reinterpret_cast<float4*>(out_plain + row * D + c) = y;
      if (out_split) {
        float4 hi, lo;
        hi.x = espb::tf32_hi(y.x); hi.y = espb::tf32_hi(y.y); hi.z = espb::tf32_hi(y.z); hi.w = espb::tf32_hi(y.w);
        lo.x = espb::tf32_lo(y.x, hi.x); lo.y = espb::tf32_lo(y.y, hi.y); lo.z = espb::tf32_lo(y.z, hi.z); lo.w = espb::tf32_lo(y.w, hi.w);
        *reinterpret_cast<float4*>(out_split + row * D + c) = hi;
        *reinterpret_cast<float4*>(out_split + split_plane + row * D + c) = lo;
      }
    }
  }
}

// ---------------------------------------------------------------- fp32 -> hi/lo planes (weights, pos-emb)
__global__ void split_kernel(const float* __restrict__ x, long long n, float* __restrict__ out, long long plane) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) store_split(out + i, plane, x[i]);
}

// ---------------------------------------------------------------- conv1: Conv2d(1, C, 3, stride 2) + ReLU (subsampling.py:400-402)
// feats [B][Tf_max][F] -> parity-split NHWC planes [B][plane*4 + (t1&1)*2 + (f1&1)][F1h][T1h][C]
// (hi/lo planes), the layout conv2's implicit GEMM reads with unit-stride TMA boxes.
__global__ void __launch_bounds__(256) conv1_relu_kernel(const float* __restrict__ feats, int Tf_max, int F, const float* __restrict__ w /*[C][9]*/,
                                                         const float* __restrict__ bias, int C, float* __restrict__ out, int T1, int F1, int T1h,
                                                         int F1h) {
  extern __shared__ float rows[];  // 3 * F input rows
  const int b = blockIdx.y, t1 = blockIdx.x;
  const float* in = feats + ((long long)b * Tf_max + 2 * t1) * F;
  for (int i = threadIdx.x; i < 3 * F; i += blockDim.x) rows[i] = in[i];
  __syncthreads();
  const long long sub = (long long)F1h * T1h * C;
  float* ob = out + (long long)b * 8 * sub;
  const int pt = t1 & 1, tt = t1 >> 1;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float wk[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) wk[i] = w[c * 9 + i];
    const float bc = bias[c];
    for (int f1 = 0; f1 < F1; ++f1) {
      float acc = bc;
#pragma unroll
      for (int kt = 0; kt < 3; ++kt)
#pragma unroll
        for (int kf = 0; kf < 3; ++kf) acc = fmaf(rows[kt * F + 2 * f1 + kf], wk[kt * 3 + kf], acc);
      acc = fmaxf(acc, 0.f);
      const int par = pt * 2 + (f1 & 1), ff = f1 >> 1;
      float* o = ob + par * sub + ((long long)ff * T1h + tt) * C + c;
      float h = tf32_hi(acc);
      o[0] = h;
      o[4 * sub] = tf32_lo(acc, h);
    }
  }
}

// ---------------------------------------------------------------- attention glue (attention.py:416-459)
// q (+bias already) lives in the split qkv buffer [M][3D] (hi/lo planes). Writes QU = q+pos_bias_u and QV = q+pos_bias_v as split [M][D].
__global__ void qu_qv_kernel(const float* __restrict__ qkv, long long qkv_plane, long long M, int D, const float* __restrict__ pos_u,
                             const float* __restrict__ pos_v, float* __restrict__ qu, float* __restrict__ qv, long long out_plane) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * D) return;
  long long r = i / D; int c = (int)(i % D);
  const float* p = qkv + r * 3 * D + c;
  float q = p[0] + p[qkv_plane];
  store_split(qu + i, out_plane, q + pos_u[c]);
  store_split(qv + i, out_plane, q + pos_v[c]);
}

// V [b][t][h*dk+d] (cols 2D.. of the split qkv buffer) -> VT split [b][h][dk][Tp]; rows t >= len_b are written as 0 so that
// zero probabilities never meet non-finite padding.
__global__ void v_transpose_kernel(const float* __restrict__ qkv, long long qkv_plane, int Tmax, int D, int H, const int* __restrict__ lens,
                                   float* __restrict__ vt, long long vt_plane, int Tp) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z / H, h = blockIdx.z % H, dk = D / H;
  const int t0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  const int len = lens[b];
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int t = t0 + i, d = d0 + threadIdx.x;
    float v = 0.f;
    if (t < len && d < dk) {
      const float* p = qkv + ((long long)b * Tmax + t) * 3 * D + 2 * D + h * dk + d;
      v = p[0] + p[qkv_plane];
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int d = d0 + i, t = t0 + threadIdx.x;
    if (d < dk && t < Tp) store_split(vt + (((long long)b * H + h) * dk + d) * Tp + t, vt_plane, tile[threadIdx.x][i]);
  }
}

// scores = (ac[i][j] + bd[i][T-1-i+j]) / sqrt(dk) (rel_shift, attention.py:391-414,455-457); keys j >= len masked
// (masked_fill(min) -> softmax -> masked_fill(0), attention.py:136-141). One warp per (b,h,i) row. Output split probs [.][Tp].
// NV > 0: the row (len <= 32*NV keys) is held in registers, so ac / bd are read exactly once; NV == 0: three-pass fallback.
template <int NV>
__global__ void __launch_bounds__(256) relpos_softmax_kernel(const float* __restrict__ ac, const float* __restrict__ bd, int B, int H, int T, int Tp,
                                                             int Rp, const int* __restrict__ lens, float inv_scale_div,
                                                             float* __restrict__ probs, long long probs_plane) {
  const long long rowid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (rowid >= (long long)B * H * T) return;
  const int lane = threadIdx.x & 31;
  const int i = (int)(rowid % T);
  const int b = (int)(rowid / ((long long)H * T));
  const int len = lens[b];
  const float* ar = ac + rowid * Tp;
  const float* br = bd + rowid * Rp + (T - 1 - i);
  float* pr = probs + rowid * Tp;
  if (NV > 0) {
    float v[NV > 0 ? NV : 1];
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int j = lane + 32 * k;
      v[k] = (j < len) ? (__ldg(ar + j) + __ldg(br + j)) / inv_scale_div : -INFINITY;
      mx = fmaxf(mx, v[k]);
    }
    mx = espb::warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      v[k] = (lane + 32 * k < len) ? expf(v[k] - mx) : 0.f;
      sum += v[k];
    }
    sum = espb::warp_sum(sum);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int j = lane + 32 * k;
      if (j < Tp) store_split(pr + j, probs_plane, v[k] / sum);
    }
    for (int j = lane + 32 * NV; j < Tp; j += 32) store_split(pr + j, probs_plane, 0.f);
    return;
  }
  float mx = -INFINITY;
  for (int j = lane; j < len; j += 32) mx = fmaxf(mx, (ar[j] + br[j]) / inv_scale_div);
  mx = espb::warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < len; j += 32) sum += expf((ar[j] + br[j]) / inv_scale_div - mx);
  sum = espb::warp_sum(sum);
  for (int j = lane; j < Tp; j += 32) {
    float p = 0.f;
    if (j < len) p = expf((ar[j] + br[j]) / inv_scale_div - mx) / sum;
    store_split(pr + j, probs_plane, p);
  }
}

// Long rows: the combined scores of a row are parked in shared memory (one row per warp), so ac / bd are read from global exactly
// once and the division / exp run once per element; ac loads and the hi/lo probability stores are 128-bit (lane owns 4 consecutive keys).
__global__ void __launch_bounds__(256) relpos_softmax_smem_kernel(const float* __restrict__ ac, const float* __restrict__ bd, int B, int H, int T, int Tp,
                                                                  int Rp, const int* __restrict__ lens, float inv_scale_div,
                                                                  float* __restrict__ probs, long long probs_plane) {
  extern __shared__ float sm_rows[];   // [8][Tp]
  const long long rowid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (rowid >= (long long)B * H * T) return;
  const int lane = threadIdx.x & 31;
  float* row = sm_rows + (threadIdx.x >> 5) * Tp;
  const int i = (int)(rowid % T);
  const int b = (int)(rowid / ((long long)H * T));
  const int len = lens[b];
  const float* ar = ac + rowid * Tp;
  const float* br = bd + rowid * Rp + (T - 1 - i);
  float* pr = probs + rowid * Tp;
  float mx = -INFINITY;
  for (int j = 4 * lane; j < len; j += 128) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(ar + j));
    float4 s;
    s.x = (a.x + __ldg(br + j)) / inv_scale_div;
    s.y = (j + 1 < len) ? (a.y + __ldg(br + j + 1)) / inv_scale_div : -INFINITY;
    s.z = (j + 2 < len) ? (a.z + __ldg(br + j + 2)) / inv_scale_div : -INFINITY;
    s.w = (j + 3 < len) ? (a.w + __ldg(br + j + 3)) / inv_scale_div : -INFINITY;
    *reinterpret_cast<float4*>(row + j) = s;
    mx = fmaxf(fmaxf(mx, s.x), fmaxf(fmaxf(s.y, s.z), s.w));
  }
  mx = espb::warp_max(mx);
  float sum = 0.f;
  for (int j = 4 * lane; j < len; j += 128) {
    float4 s = *reinterpret_cast<const float4*>(row + j);
    s.x = expf(s.x - mx);
    s.y = (j + 1 < len) ? expf(s.y - mx) : 0.f;
    s.z = (j + 2 < len) ? expf(s.z - mx) : 0.f;
    s.w = (j + 3 < len) ? expf(s.w - mx) : 0.f;
    *reinterpret_cast<float4*>(row + j) = s;
    sum += (s.x + s.y) + (s.z + s.w);
  }
  sum = espb::warp_sum(sum);
  for (int j = 4 * lane; j < Tp; j += 128) {
    float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
    if (j < len) e = *reinterpret_cast<const float4*>(row + j);
    float4 hi, lo;
    const float p0 = e.x / sum, p1 = e.y / sum, p2 = e.z / sum, p3 = e.w / sum;
    hi.x = espb::tf32_hi(p0); hi.y = espb::tf32_hi(p1); hi.z = espb::tf32_hi(p2); hi.w = espb::tf32_hi(p3);
    lo.x = espb::tf32_lo(p0, hi.x); lo.y = espb::tf32_lo(p1, hi.y); lo.z = espb::tf32_lo(p2, hi.z); lo.w = espb::tf32_lo(p3, hi.w);
    *reinterpret_cast<float4*>(pr + j) = hi;
    *reinterpret_cast<float4*>(pr + probs_plane + j) = lo;
  }
}

// Plain (absolute-position) attention: scores / sqrt(d_k), keys >= len masked, softmax, masked again (attention.py:121-151, 262-265).
// One warp per (b, h, query) row, three passes over the row (the rows are short-lived L1 / L2 residents).  Output split probs [.][Tp].
__global__ void __launch_bounds__(256) masked_softmax_kernel(const float* __restrict__ sc, int B, int H, int T, int Tp, const int* __restrict__ lens,
                                                             float scale_div, float* __restrict__ probs, long long probs_plane) {
  const long long rowid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (rowid >= (long long)B * H * T) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(rowid / ((long long)H * T));
  const int len = lens[b];
  const float* ar = sc + rowid * Tp;
  float* pr = probs + rowid * Tp;
  float mx = -INFINITY;
  for (int j = lane; j < len; j += 32) mx = fmaxf(mx, ar[j] / scale_div);
  mx = espb::warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < len; j += 32) sum += expf(ar[j] / scale_div - mx);
  sum = espb::warp_sum(sum);
  for (int j = lane; j < Tp; j += 32) {
    float p = 0.f;
    if (j < len) p = expf(ar[j] / scale_div - mx) / sum;
    store_split(pr + j, probs_plane, p);
  }
}

// ---------------------------------------------------------------- convolution module (convolution.py:56-79)
// y [M][2C] = pointwise_conv1 output. GLU -> depthwise conv (K taps, zero pad at the utterance's own ends) ->
// BatchNorm eval folded to x*bn_a + bn_b -> Swish -> split [M][C].
constexpr int DW_TT = 64, DW_CC = 64;
__global__ void __launch_bounds__(256) glu_dwconv_bn_swish_kernel(const float* __restrict__ y, int Tmax, int C, const int* __restrict__ lens,
                                                                  const float* __restrict__ dw_w /*[C][K]*/, const float* __restrict__ dw_b, int K,
                                                                  const float* __restrict__ bn_a, const float* __restrict__ bn_b,
                                                                  float* __restrict__ out, long long out_plane) {
  extern __shared__ float sm[];  // [(DW_TT + K - 1)][DW_CC] GLU'd tile, then [DW_CC][K] weights
  const int b = blockIdx.z, t0 = blockIdx.x * DW_TT, c0 = blockIdx.y * DW_CC;
  const int len = lens[b], pad = (K - 1) / 2, rows = DW_TT + K - 1;
  float* tile = sm;
  float* wts = sm + rows * DW_CC;
  for (int i = threadIdx.x; i < rows * DW_CC; i += blockDim.x) {
    int r = i / DW_CC, c = c0 + (i % DW_CC), t = t0 - pad + r;
    float v = 0.f;
    if (t >= 0 && t < len && c < C) {
      const float* p = y + ((long long)b * Tmax + t) * 2 * C;
      float a = p[c], g = p[C + c];
      v = a * (1.f / (1.f + expf(-g)));
    }
    tile[i] = v;
  }
  for (int i = threadIdx.x; i < DW_CC * K; i += blockDim.x) {
    int c = c0 + i / K;
    wts[i] = (c < C) ? dw_w[(long long)c * K + (i % K)] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < DW_TT * DW_CC; i += blockDim.x) {
    int tl = i / DW_CC, cl = i % DW_CC, t = t0 + tl, c = c0 + cl;
    if (t >= Tmax || c >= C) continue;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) acc = fmaf(tile[(tl + k) * DW_CC + cl], wts[cl * K + k], acc);
    acc += dw_b[c];
    float z = acc * bn_a[c] + bn_b[c];
    z = espb::swish_acc(z);
    if (t >= len) z = 0.f;
    store_split(out + ((long long)b * Tmax + t) * C + c, out_plane, z);
  }
}

// Same arithmetic (per output the same fmaf chain over k = 0..K-1, so bit-identical results), sliding window in registers: a thread owns one
// channel and DW_RUN consecutive frames, reads each of the DW_RUN + K - 1 GLU'd inputs of its column once from shared memory and feeds it to the
// up to K outputs it belongs to -- 2.9 shared-memory loads per output instead of 2 K (the first kernel is LDS-bound: 62 loads per output at K = 31).
constexpr int DW_RUN = 16;
template <int K>
__global__ void __launch_bounds__(256) glu_dwconv_bn_swish_win_kernel(const float* __restrict__ y, int Tmax, int C, const int* __restrict__ lens,
                                                                      const float* __restrict__ dw_w /*[C][K]*/, const float* __restrict__ dw_b,
                                                                      const float* __restrict__ bn_a, const float* __restrict__ bn_b,
                                                                      float* __restrict__ out, long long out_plane) {
  static_assert(DW_TT == 4 * DW_RUN && DW_CC == 64, "256 threads = 64 channels x 4 runs of DW_RUN frames");
  extern __shared__ float sm[];  // [(DW_TT + K - 1)][DW_CC] GLU'd tile
  const int b = blockIdx.z, t0 = blockIdx.x * DW_TT, c0 = blockIdx.y * DW_CC;
  const int len = lens[b];
  constexpr int pad = (K - 1) / 2, rows = DW_TT + K - 1;
  for (int i = threadIdx.x; i < rows * DW_CC; i += blockDim.x) {
    const int r = i / DW_CC, c = c0 + (i % DW_CC), t = t0 - pad + r;
    float v = 0.f;
    if (t >= 0 && t < len && c < C) {
      const float* p = y + ((long long)b * Tmax + t) * 2 * C;
      const float a = p[c], g = p[C + c];
      v = a * (1.f / (1.f + expf(-g)));
    }
    sm[i] = v;
  }
  __syncthreads();
  const int cl = threadIdx.x & 63, run = threadIdx.x >> 6, c = c0 + cl;
  if (c >= C) return;
  float w[K];
#pragma unroll
  for (int k = 0; k < K; ++k) w[k] = __ldg(dw_w + (long long)c * K + k);
  float acc[DW_RUN];
#pragma unroll
  for (int o = 0; o < DW_RUN; ++o) acc[o] = 0.f;
  const float* col = sm + (run * DW_RUN) * DW_CC + cl;
#pragma unroll
  for (int r = 0; r < DW_RUN + K - 1; ++r) {
    const float x = col[r * DW_CC];
#pragma unroll
    for (int o = 0; o < DW_RUN; ++o) {
      if (r - o >= 0 && r - o < K) acc[o] = fmaf(x, w[r - o], acc[o]);   // resolved at compile time: input r is tap r - o of output o
    }
  }
  const float db = dw_b[c], ba = bn_a[c], bb = bn_b[c];
#pragma unroll
  for (int o = 0; o < DW_RUN; ++o) {
    const int t = t0 + run * DW_RUN + o;
    if (t >= Tmax) break;
    float z = (acc[o] + db) * ba + bb;
    z = espb::swish_acc(z);
    if (t >= len) z = 0.f;
    store_split(out + ((long long)b * Tmax + t) * C + c, out_plane, z);
  }
}

// x[b, t >= len_b, :] = 0 for plain and split buffers (keeps padded rows finite).
__global__ void zero_pad_rows_kernel(float* __restrict__ x, int Tmax, int D, const int* __restrict__ lens, long long plane, int nplanes) {
  const int b = blockIdx.y;
  const int len = lens[b];
  long long n = (long long)(Tmax - len) * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float* p = x + ((long long)b * Tmax + len) * D + i;
    for (int q = 0; q < nplanes; ++q) p[q * plane] = 0.f;
  }
}

// ---------------------------------------------------------------- contextual block processing (streaming encoder, SURVEY 8f-2)
// contextual_block_conformer_encoder.py:506-541: blocks of `block` frames every `hop` frames, framed by two context tokens:
//   chunk[n][i][0]          = context vector of the previous block (or of the previous call / of this block for the very first one)
//   chunk[n][i][1..len]     = pos_enc(xs[n][i*hop + t], start pos0 + i*hop)        (StreamPositionalEncoding: x * sqrt(D) + pe[pos])
//   chunk[n][i][block+1]    = addin_i = pos_enc(mean_t xs[n][i*hop .. +len), start ctx0 + i)
// rows len+1..block of a trailing partial block stay zero.
__global__ void __launch_bounds__(128) cbe_build_chunks_kernel(const float* __restrict__ xs, int Tt, int D, int nb, int block, int hop,
                                                               const float* __restrict__ pe, int pos0, int ctx0, float scale,
                                                               const float* __restrict__ prev_addin, float* __restrict__ addin_out,
                                                               float* __restrict__ chunks) {
  const int i = blockIdx.x, n = blockIdx.y, S = block + 2;
  const float* x = xs + (long long)n * Tt * D;
  float* c = chunks + ((long long)n * nb + i) * S * D;
  const int cur = i * hop, len = min(block, Tt - cur);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float sum = 0.f;
    for (int t = 0; t < len; ++t) {
      const float v = x[(long long)(cur + t) * D + d];
      sum += v;
      c[(long long)(1 + t) * D + d] = v * scale + pe[(long long)(pos0 + cur + t) * D + d];
    }
    for (int t = len; t < block; ++t) c[(long long)(1 + t) * D + d] = 0.f;
    const float addin = (sum / (float)len) * scale + pe[(long long)(ctx0 + i) * D + d];
    c[(long long)(block + 1) * D + d] = addin;
    float prev;
    if (i > 0) {
      const int pc = (i - 1) * hop, pl = min(block, Tt - pc);
      float ps = 0.f;
      for (int t = 0; t < pl; ++t) ps += x[(long long)(pc + t) * D + d];
      prev = (ps / (float)pl) * scale + pe[(long long)(ctx0 + i - 1) * D + d];
    } else {
      prev = prev_addin ? prev_addin[(long long)n * D + d] : addin;
    }
    c[d] = prev;
    if (i == nb - 1) addin_out[(long long)n * D + d] = addin;
  }
}

// contextual_block_encoder_layer.py:291-308: after a layer, token 0 of every block becomes the previous block's last token (the context
// inherited from the layer below it in time); the first block takes the context kept from the previous call; the last one is kept.
__global__ void __launch_bounds__(128) cbe_ctx_propagate_kernel(float* __restrict__ x, int nb, int S, int D, const float* __restrict__ past_ctx,
                                                                float* __restrict__ next_ctx, int layer, int L) {
  const int i = blockIdx.x, n = blockIdx.y;
  float* xb = x + ((long long)n * nb + i) * S * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float v;
    if (i > 0) v = xb[-(long long)S * D + (long long)(S - 1) * D + d];                   // last token of block i-1
    else v = past_ctx ? past_ctx[((long long)n * L + layer) * D + d] : xb[(long long)(S - 1) * D + d];
    if (i == nb - 1) next_ctx[((long long)n * L + layer) * D + d] = xb[(long long)(S - 1) * D + d];
    xb[d] = v;          // token 0; every value read above is a LAST token, which nobody writes
  }
}

// rows row0 + k * every (k < count) of a [rows][D] buffer (nplanes planes) := 0
__global__ void zero_rows_kernel(float* __restrict__ x, long long row0, long long every, long long count, int D, long long plane, int nplanes) {
  const long long k = blockIdx.x;
  if (k >= count) return;
  float* r = x + (row0 + k * every) * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x)
    for (int q = 0; q < nplanes; ++q) r[q * plane + d] = 0.f;
}

// out[n][t][:] = src[n][idx[t]][:]
__global__ void gather_rows_kernel(const float* __restrict__ src, long long src_rows, const int* __restrict__ idx, int nout, int D,
                                   float* __restrict__ out) {
  const int t = blockIdx.x, n = blockIdx.y;
  const float* s = src + ((long long)n * src_rows + idx[t]) * D;
  float* o = out + ((long long)n * nout + t) * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) o[d] = s[d];
}

}  // namespace

extern "C" {

int espb_cbe_build_chunks_f32(const float* xs, int N, int Tt, int D, int nb, int block, int hop, const float* pe, int pos0, int ctx0, float scale,
                              const float* prev_addin, float* addin_out, float* chunks, cudaStream_t stream) {
  if (N <= 0 || nb <= 0 || block <= 0 || hop <= 0 || (nb - 1) * hop >= Tt) { espb_set_error("cbe_build_chunks: bad shape"); return ESPB_ERR_ARG; }
  cbe_build_chunks_kernel<<<dim3(nb, N), 128, 0, stream>>>(xs, Tt, D, nb, block, hop, pe, pos0, ctx0, scale, prev_addin, addin_out, chunks);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_cbe_ctx_propagate_f32(float* x, int N, int nb, int S, int D, const float* past_ctx, float* next_ctx, int layer, int L,
                               cudaStream_t stream) {
  if (N <= 0 || nb <= 0) return ESPB_OK;
  // block i reads the last token of block i-1, which no block writes (only tokens 0 are written): one launch is race-free
  cbe_ctx_propagate_kernel<<<dim3(nb, N), 128, 0, stream>>>(x, nb, S, D, past_ctx, next_ctx, layer, L);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_zero_rows_f32(float* x, long long row0, long long every, long long count, int D, long long plane, int nplanes, cudaStream_t stream) {
  if (count <= 0) return ESPB_OK;
  zero_rows_kernel<<<(unsigned)count, 128, 0, stream>>>(x, row0, every, count, D, plane, nplanes);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_gather_rows_f32(const float* src, int N, long long src_rows, const int* idx, int nout, int D, float* out, cudaStream_t stream) {
  if (N <= 0 || nout <= 0) return ESPB_OK;
  gather_rows_kernel<<<dim3(nout, N), 128, 0, stream>>>(src, src_rows, idx, nout, D, out);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_layernorm_f32(const float* x, long long rows, int D, const float* gamma, const float* beta, float eps, float* out_plain,
                       float* out_split, long long split_plane, cudaStream_t stream) {
  if (D > 2048 || D <= 0) { espb_set_error("layernorm: D must be in (0, 2048]"); return ESPB_ERR_ARG; }
  if (rows <= 0) return ESPB_OK;
  {
    const uintptr_t al = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta) |
                         reinterpret_cast<uintptr_t>(out_plain) | reinterpret_cast<uintptr_t>(out_split);
    if ((D & 3) == 0 && D <= 1024 && (al & 15) == 0 && (split_plane & 3) == 0 && !getenv("ESPB_LN_SCALAR")) {
      const int rpb = rows <= 4096 ? 2 : 8;   // rows (warps) per block
      const dim3 g((unsigned)((rows + rpb - 1) / rpb)), blk(32 * rpb);
      if (D <= 256) espb::launch_pdl(layernorm_vec_kernel<2>, g, blk, 0, stream, x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane);
      else if (D <= 512) espb::launch_pdl(layernorm_vec_kernel<4>, g, blk, 0, stream, x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane);
      else espb::launch_pdl(layernorm_vec_kernel<8>, g, blk, 0, stream, x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane);
      ESPB_CHECK_LAUNCH();
      return ESPB_OK;
    }
  }
  const unsigned grid = (unsigned)((rows + 7) / 8);
  if (D <= 256) espb::launch_pdl(layernorm_kernel<8>, dim3(grid), dim3(256), 0, stream, x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane);
  else if (D <= 512) espb::launch_pdl(layernorm_kernel<16>, dim3(grid), dim3(256), 0, stream, x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane);
  else if (D <= 1024) espb::launch_pdl(layernorm_kernel<32>, dim3(grid), dim3(256), 0, stream, x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane);
  else espb::launch_pdl(layernorm_kernel<64>, dim3(grid), dim3(256), 0, stream, x, rows, D, gamma, beta, eps, out_plain, out_split, split_plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_split_tf32_f32(const float* x, long long n, float* out, long long plane, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  split_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(x, n, out, plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_conv1_relu_f32(const float* feats, int B, int Tf_max, int F, const float* w, const float* bias, int C, float* out, int T1, int F1,
                        int T1h, int F1h, cudaStream_t stream) {
  if (T1 <= 0 || F1 <= 0) { espb_set_error("conv1: empty output"); return ESPB_ERR_ARG; }
  dim3 grid(T1, B);
  conv1_relu_kernel<<<grid, 256, 3 * F * sizeof(float), stream>>>(feats, Tf_max, F, w, bias, C, out, T1, F1, T1h, F1h);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_qu_qv_f32(const float* qkv, long long qkv_plane, long long M, int D, const float* pos_u, const float* pos_v, float* qu, float* qv,
                   long long out_plane, cudaStream_t stream) {
  long long n = M * D;
  qu_qv_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(qkv, qkv_plane, M, D, pos_u, pos_v, qu, qv, out_plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_v_transpose_f32(const float* qkv, long long qkv_plane, int B, int Tmax, int D, int H, const int* lens, float* vt, long long vt_plane,
                         int Tp, cudaStream_t stream) {
  const int dk = D / H;
  dim3 grid((Tp + 31) / 32, (dk + 31) / 32, B * H), block(32, 8);
  v_transpose_kernel<<<grid, block, 0, stream>>>(qkv, qkv_plane, Tmax, D, H, lens, vt, vt_plane, Tp);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_relpos_softmax_f32(const float* ac, const float* bd, int B, int H, int T, int Tp, int Rp, const int* lens, float sqrt_dk, float* probs,
                            long long probs_plane, cudaStream_t stream) {
  long long rows = (long long)B * H * T;
  const unsigned grid = (unsigned)((rows + 7) / 8);
  // (a register-resident single-pass variant <NV> has lower occupancy; kept for short rows)
  if (T <= 128) relpos_softmax_kernel<4><<<grid, 256, 0, stream>>>(ac, bd, B, H, T, Tp, Rp, lens, sqrt_dk, probs, probs_plane);
  else if ((Tp & 3) == 0 && (probs_plane & 3) == 0 && (reinterpret_cast<uintptr_t>(ac) & 15) == 0 && (reinterpret_cast<uintptr_t>(probs) & 15) == 0 &&
           (size_t)8 * Tp * sizeof(float) <= 48 * 1024 && !getenv("ESPB_SOFTMAX_3PASS"))
    relpos_softmax_smem_kernel<<<grid, 256, (size_t)8 * Tp * sizeof(float), stream>>>(ac, bd, B, H, T, Tp, Rp, lens, sqrt_dk, probs, probs_plane);
  else relpos_softmax_kernel<0><<<grid, 256, 0, stream>>>(ac, bd, B, H, T, Tp, Rp, lens, sqrt_dk, probs, probs_plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_masked_softmax_f32(const float* scores, int B, int H, int T, int Tp, const int* lens, float sqrt_dk, float* probs, long long probs_plane,
                            cudaStream_t stream) {
  const long long rows = (long long)B * H * T;
  masked_softmax_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(scores, B, H, T, Tp, lens, sqrt_dk, probs, probs_plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_glu_dwconv_bn_swish_f32(const float* y, int B, int Tmax, int C, const int* lens, const float* dw_w, const float* dw_b, int K,
                                 const float* bn_a, const float* bn_b, float* out, long long out_plane, cudaStream_t stream) {
  if (K < 1 || (K & 1) == 0 || K > 127) { espb_set_error("dwconv: kernel size must be odd and <= 127"); return ESPB_ERR_ARG; }
  dim3 grid((Tmax + DW_TT - 1) / DW_TT, (C + DW_CC - 1) / DW_CC, B);
  static int v1 = -1;
  if (v1 < 0) v1 = getenv("ESPB_DWCONV_V1") ? 1 : 0;
  const size_t smem_win = (size_t)(DW_TT + K - 1) * DW_CC * sizeof(float);
  if (!v1 && K == 31) {
    glu_dwconv_bn_swish_win_kernel<31><<<grid, 256, smem_win, stream>>>(y, Tmax, C, lens, dw_w, dw_b, bn_a, bn_b, out, out_plane);
  } else if (!v1 && K == 15) {
    glu_dwconv_bn_swish_win_kernel<15><<<grid, 256, smem_win, stream>>>(y, Tmax, C, lens, dw_w, dw_b, bn_a, bn_b, out, out_plane);
  } else {
    const size_t smem = ((size_t)(DW_TT + K - 1) * DW_CC + (size_t)DW_CC * K) * sizeof(float);
    glu_dwconv_bn_swish_kernel<<<grid, 256, smem, stream>>>(y, Tmax, C, lens, dw_w, dw_b, K, bn_a, bn_b, out, out_plane);
  }
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_zero_pad_rows_f32(float* x, int B, int Tmax, int D, const int* lens, long long plane, int nplanes, cudaStream_t stream) {
  dim3 grid(32, B);
  zero_pad_rows_kernel<<<grid, 256, 0, stream>>>(x, Tmax, D, lens, plane, nplanes);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

}  // extern "C"
