// RNN ASR model family (espnet2/asr/encoder/vgg_rnn_encoder.py, rnn_encoder.py, asr/decoder/rnn_decoder.py): the VGG2L glue around its
// implicit-GEMM convs, the step of the (bi)LSTM recurrence, the projection epilogue and the location-aware attention step of the decoder.
// Every GEMM of the family (VGG convs, input-to-gate products, h W_hh^T, projections, mlp_enc / mlp_dec, decoder gates and output) runs on
// espb_gemm_f32; these kernels are the element-wise and per-slot work between them.
#include "common.cuh"
#include "../../include/espnet_b200.h"

namespace {

__device__ __forceinline__ void store_split(float* p, long long plane, float v) {
  const float hi = espb::tf32_hi(v);
  p[0] = hi;
  p[plane] = espb::tf32_lo(v, hi);
}

// conv1_1 (Conv2d(1, C, 3, 1, 1)) + ReLU over the (time, freq) plane of utterance b, which sees zeros at t >= lens[b].  Output: the
// zero-bordered split input of the next implicit-GEMM conv, [B][2][F + 2][T + 2][C]; rows t >= lens[b] and the border are 0.
__global__ void vgg_conv1_kernel(const float* __restrict__ feats, int Tf_max, int F, const int* __restrict__ lens, const float* __restrict__ w,
                                 const float* __restrict__ bias, int C, float* __restrict__ out, int T) {
  const int Fp = F + 2, Tp = T + 2;
  const int b = blockIdx.z, fp = blockIdx.y;
  const int tp = blockIdx.x * (blockDim.x / C) + threadIdx.x / C, c = threadIdx.x % C;
  if (tp >= Tp || threadIdx.x >= (blockDim.x / C) * C) return;
  const int len = lens[b], t = tp - 1, f = fp - 1;
  float v = 0.f;
  if (t >= 0 && t < len && f >= 0 && f < F) {
    const float* x = feats + (long long)b * Tf_max * F;
    float acc = 0.f;
#pragma unroll
    for (int kt = 0; kt < 3; ++kt) {
      const int ti = t + kt - 1;
      if (ti < 0 || ti >= len) continue;
#pragma unroll
      for (int kf = 0; kf < 3; ++kf) {
        const int fi = f + kf - 1;
        if (fi < 0 || fi >= F) continue;
        acc = fmaf(w[c * 9 + kt * 3 + kf], x[(long long)ti * F + fi], acc);
      }
    }
    v = fmaxf(acc + bias[c], 0.f);
  }
  const long long plane = (long long)Fp * Tp * C;
  store_split(out + (long long)b * 2 * plane + ((long long)fp * Tp + tp) * C + c, plane, v);
}

// Conv output x [B][F][T][C] (plain, ReLU applied) of utterance b, valid at t < lens[b] -> (pool: 2x2 max-pool, ceil mode, over the valid
// rows only) -> flat = 0: the zero-bordered split input of the next conv [B][2][Fo + 2][To + 2][C], rows t >= the new length zero;
// flat = 1: split rows [B * To][C * Fo] in the reference's (channel, freq) flattening, rows t >= the new length zero.
__global__ void vgg_pool_kernel(const float* __restrict__ x, int F, int T, int C, const int* __restrict__ lens, int pool, int flat,
                                float* __restrict__ out, long long out_plane) {
  const int Fo = pool ? (F + 1) / 2 : F, To = pool ? (T + 1) / 2 : T;
  const int b = blockIdx.z;
  const int len = lens[b], olen = pool ? (len + 1) / 2 : len;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int FoE = flat ? Fo : Fo + 2, ToE = flat ? To : To + 2;
  if (i >= (long long)FoE * ToE * C) return;
  const int c = flat ? (int)((i / Fo) % C) : (int)(i % C);   // flat: fo fastest, so that neighbouring threads write neighbouring columns
  int fo, to;
  if (flat) { fo = (int)(i % Fo); to = (int)(i / ((long long)C * Fo)); }
  else { to = (int)((i / C) % ToE) - 1; fo = (int)(i / ((long long)C * ToE)) - 1; }
  float v = 0.f;
  if (to >= 0 && to < olen && fo >= 0 && fo < Fo) {
    const float* xb = x + (long long)b * F * T * C;
    if (pool) {
      v = -INFINITY;
      for (int df = 0; df < 2; ++df)
        for (int dt = 0; dt < 2; ++dt) {
          const int f = 2 * fo + df, t = 2 * to + dt;
          if (f < F && t < len) v = fmaxf(v, xb[((long long)f * T + t) * C + c]);
        }
    } else {
      v = xb[((long long)fo * T + to) * C + c];
    }
  }
  if (flat) store_split(out + ((long long)b * To + to) * C * Fo + (long long)c * Fo + fo, out_plane, v);
  else store_split(out + (long long)b * 2 * out_plane + i, out_plane, v);
}

__device__ __forceinline__ float sigmoid_acc(float v) { return 1.f / (1.f + expf(-v)); }

// Step s of a 1-layer (B)LSTM over B utterances: direction d of utterance b handles frame t = s (d = 0) or lens[b] - 1 - s (d = 1).
// gates = xg[b][t][d * 4H ..] (input product + both biases) + hg[d][b][..] (h_{t-1} W_hh^T; absent at s = 0, where h and c start at 0).
// h' -> h split [2][ndir][B][Hp] (the next step's GEMM operand) and y split [B][T][ldy] at columns d * H ..; c' -> c [ndir][B][H].
// At s >= lens[b], y[b][s] of both directions is set to 0 (the padded frames of pad_packed_sequence).
__global__ void lstm_rec_kernel(const float* __restrict__ xg, const float* __restrict__ hg, const int* __restrict__ lens, int s, int B, int T,
                                int H, int Hp, int ndir, float* __restrict__ h, long long h_plane, float* __restrict__ c, float* __restrict__ y,
                                long long y_plane, int ldy) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)ndir * B * H) return;
  const int j = (int)(i % H), b = (int)((i / H) % B), d = (int)(i / ((long long)H * B));
  const int len = lens[b];
  if (s >= len) {
    if (s < T) store_split(y + ((long long)b * T + s) * ldy + d * H + j, y_plane, 0.f);
    return;
  }
  const int t = d ? len - 1 - s : s;
  const float* g = xg + ((long long)b * T + t) * ndir * 4 * H + (long long)d * 4 * H + j;
  float gi = g[0], gf = g[H], gg = g[2 * H], go = g[3 * H];
  float cp = 0.f;
  const long long sidx = ((long long)d * B + b);
  if (s > 0) {
    const float* r = hg + sidx * 4 * H + j;
    gi += r[0]; gf += r[H]; gg += r[2 * H]; go += r[3 * H];
    cp = c[sidx * H + j];
  }
  const float cn = sigmoid_acc(gf) * cp + sigmoid_acc(gi) * tanhf(gg);
  const float hn = sigmoid_acc(go) * tanhf(cn);
  c[sidx * H + j] = cn;
  store_split(h + sidx * Hp + j, h_plane, hn);
  store_split(y + ((long long)b * T + t) * ldy + d * H + j, y_plane, hn);
}

// Projection epilogue: x [B][T][D] (plain, row stride D) -> v = tanh(x) (act) or x, rows t >= lens[b] set to 0; v into x in place
// (write_plain) and/or split into out [B*T][ldo] (out may be NULL).
__global__ void rnn_proj_post_kernel(float* __restrict__ x, int B, int T, int D, const int* __restrict__ lens, int act, int write_plain,
                                     float* __restrict__ out, long long out_plane, int ldo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * T * D) return;
  const int d = (int)(i % D);
  const long long row = i / D;
  const int t = (int)(row % T), b = (int)(row / T);
  float v = t < lens[b] ? x[i] : 0.f;
  if (act) v = tanhf(v);
  if (t >= lens[b]) v = 0.f;
  if (write_plain) x[i] = v;
  if (out) store_split(out + row * ldo + d, out_plane, v);
}

// AttLoc (legacy/nets/pytorch_backend/rnn/attentions.py:249-378) for slot s of utterance u = s / W at decoding position pos:
//   prev = ring[(pos-1)&1][anc[s][pos-1]] (pos 0: uniform 1/len), conv[c][t] = sum_k conv_w[c][k] prev[t + k - filts] (zeros outside),
//   e[t] = gvec . tanh(att_wt^T conv[:, t] + enc_h[u][t] + dec_z[s]) + gvec_b for t < len, w = softmax(2 e) over t < len,
//   ring[pos&1][s] = w (0 at t >= len), ctx = sum_t w[t] enc[u][t] split into out (and out2).
// enc is read from its split copy (hi + lo).  One block per slot; shared memory: prev (Tmax + 2 filts), conv (chans * Tmax), e (Tmax),
// att_wt (chans * A).
constexpr int ATT_THREADS = 256;
__global__ void __launch_bounds__(ATT_THREADS) att_loc_kernel(
    const float* __restrict__ enc_h, const float* __restrict__ enc, long long enc_plane, const int* __restrict__ lens, int W, int Tmax, int A,
    int E, const float* __restrict__ dec_z, const float* __restrict__ conv_w, int chans, int filts, const float* __restrict__ att_wt,
    const float* __restrict__ gvec, const float* __restrict__ gvec_b, const int* __restrict__ anc, int anc_ld, int pos,
    const int* __restrict__ step_ptr, float* __restrict__ ring, int n, float* __restrict__ out, long long out_plane, int out_ld,
    float* __restrict__ out2, long long out2_plane, int out2_ld) {
  extern __shared__ float sm[];
  __shared__ float red[33];
  const int K = 2 * filts + 1;
  float* prev = sm;                        // Tmax + 2 filts
  float* conv = prev + Tmax + 2 * filts;   // chans * Tmax
  float* e = conv + (long long)chans * Tmax;   // Tmax
  float* wt = e + Tmax;                    // chans * A
  espb::pdl_trigger();
  espb::pdl_wait();
  if (step_ptr) pos += *step_ptr;
  const int s = blockIdx.x, u = s / W, len = lens[u];
  const int p = pos > 0 ? anc[(long long)s * anc_ld + pos - 1] : -1;
  const float* rp = ring + ((long long)((pos - 1) & 1) * n + (p < 0 ? 0 : p)) * Tmax;
  for (int i = threadIdx.x; i < Tmax + 2 * filts; i += blockDim.x) {
    const int t = i - filts;
    prev[i] = (t < 0 || t >= len) ? 0.f : (p < 0 ? 1.f / (float)len : rp[t]);
  }
  for (int i = threadIdx.x; i < chans * A; i += blockDim.x) wt[i] = att_wt[i];
  __syncthreads();
  for (int i = threadIdx.x; i < chans * len; i += blockDim.x) {
    const int c = i / len, t = i % len;
    const float* wc = conv_w + (long long)c * K;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) acc = fmaf(wc[k], prev[t + k], acc);
    conv[c * Tmax + t] = acc;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* eh = enc_h + (long long)u * Tmax * A;
  const float* dz = dec_z + (long long)s * A;
  const float gb = gvec_b[0];
  for (int t = warp; t < len; t += nw) {
    float acc = 0.f;
    for (int a = lane; a < A; a += 32) {
      float loc = 0.f;
      for (int c = 0; c < chans; ++c) loc = fmaf(wt[c * A + a], conv[c * Tmax + t], loc);
      acc = fmaf(gvec[a], tanhf(loc + eh[(long long)t * A + a] + dz[a]), acc);
    }
    acc = espb::warp_sum(acc);
    if (lane == 0) e[t] = 2.f * (acc + gb);
  }
  __syncthreads();
  float m = -INFINITY;
  for (int t = threadIdx.x; t < len; t += blockDim.x) m = fmaxf(m, e[t]);
  m = espb::block_max(m, red);
  float sum = 0.f;
  for (int t = threadIdx.x; t < len; t += blockDim.x) {
    const float v = expf(e[t] - m);
    e[t] = v;
    sum += v;
  }
  sum = espb::block_sum(sum, red);
  const float inv = 1.f / sum;
  float* wr = ring + ((long long)(pos & 1) * n + s) * Tmax;
  for (int t = threadIdx.x; t < Tmax; t += blockDim.x) {
    const float v = t < len ? e[t] * inv : 0.f;
    if (t < len) e[t] = v;
    wr[t] = v;
  }
  __syncthreads();
  const float* eu = enc + (long long)u * Tmax * E;
  for (int j = threadIdx.x; j < E; j += blockDim.x) {
    float acc = 0.f;
    for (int t = 0; t < len; ++t) acc = fmaf(e[t], eu[(long long)t * E + j] + eu[enc_plane + (long long)t * E + j], acc);
    store_split(out + (long long)s * out_ld + j, out_plane, acc);
    if (out2) store_split(out2 + (long long)s * out2_ld + j, out2_plane, acc);
  }
}

__global__ void drop_cand_kernel(int* __restrict__ valid, int n, int PC, int j) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) valid[(long long)s * PC + j] = 0;
}

size_t att_smem(int Tmax, int A, int chans, int filts) {
  return sizeof(float) * ((size_t)Tmax + 2 * filts + (size_t)chans * Tmax + Tmax + (size_t)chans * A);
}

}  // namespace

extern "C" {

int espb_vgg_conv1_relu_f32(const float* feats, int B, int Tf_max, int F, const int* lens, const float* w, const float* bias, int C, float* out,
                            int T, cudaStream_t stream) {
  if (B <= 0) return ESPB_OK;
  if (C <= 0 || C > 256 || T > Tf_max || F <= 0) { espb_set_error("vgg_conv1_relu: need 0 < C <= 256, T <= Tf_max, F > 0"); return ESPB_ERR_ARG; }
  const int per = 256 / C;
  dim3 grid((unsigned)((T + 2 + per - 1) / per), (unsigned)(F + 2), (unsigned)B);
  vgg_conv1_kernel<<<grid, 256, 0, stream>>>(feats, Tf_max, F, lens, w, bias, C, out, T);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_vgg_pool_f32(const float* x, int B, int F, int T, int C, const int* lens, int pool, int flat, float* out, long long out_plane,
                      cudaStream_t stream) {
  if (B <= 0) return ESPB_OK;
  if (F <= 0 || T <= 0 || C <= 0) { espb_set_error("vgg_pool: need F, T, C > 0"); return ESPB_ERR_ARG; }
  const int Fo = pool ? (F + 1) / 2 : F, To = pool ? (T + 1) / 2 : T;
  const long long tot = (long long)(flat ? Fo : Fo + 2) * (flat ? To : To + 2) * C;
  dim3 grid((unsigned)((tot + 255) / 256), 1, (unsigned)B);
  vgg_pool_kernel<<<grid, 256, 0, stream>>>(x, F, T, C, lens, pool, flat, out, out_plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_lstm_rec_step_f32(const float* xg, const float* hg, const int* lens, int s, int B, int T, int H, int Hp, int ndir, float* h,
                           long long h_plane, float* c, float* y, long long y_plane, int ldy, cudaStream_t stream) {
  if (B <= 0) return ESPB_OK;
  if (H > Hp || (ndir != 1 && ndir != 2) || ldy < ndir * H || s < 0) {
    espb_set_error("lstm_rec_step: need H <= Hp, ndir 1 or 2, ldy >= ndir * H, s >= 0");
    return ESPB_ERR_ARG;
  }
  const long long tot = (long long)ndir * B * H;
  lstm_rec_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(xg, hg, lens, s, B, T, H, Hp, ndir, h, h_plane, c, y, y_plane, ldy);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_rnn_proj_post_f32(float* x, int B, int T, int D, const int* lens, int act, int write_plain, float* out, long long out_plane, int ldo,
                           cudaStream_t stream) {
  if (B <= 0 || T <= 0) return ESPB_OK;
  if (out && ldo < D) { espb_set_error("rnn_proj_post: need ldo >= D"); return ESPB_ERR_ARG; }
  const long long tot = (long long)B * T * D;
  rnn_proj_post_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(x, B, T, D, lens, act, write_plain, out, out_plane, ldo);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_att_loc_step_f32(const float* enc_h, const float* enc, long long enc_plane, const int* lens, int W, int Tmax, int A, int E,
                          const float* dec_z, const float* conv_w, int chans, int filts, const float* att_wt, const float* gvec,
                          const float* gvec_b, const int* anc, int anc_ld, int pos, const int* step_ptr, float* ring, int n, float* out,
                          long long out_plane, int out_ld, float* out2, long long out2_plane, int out2_ld, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  if (W <= 0 || n % W || Tmax <= 0 || A <= 0 || E <= 0 || chans <= 0 || filts < 0 || out_ld < E || (out2 && out2_ld < E)) {
    espb_set_error("att_loc_step: need W > 0 dividing n, Tmax, A, E, chans > 0, filts >= 0, out_ld (out2_ld) >= E");
    return ESPB_ERR_ARG;
  }
  const size_t smem = att_smem(Tmax, A, chans, filts);
  if (smem + 33 * sizeof(float) > 227 * 1024) {   // dynamic plus the static reduction buffer
    espb_set_error("att_loc_step: Tmax * (chans + 2) + chans * A too large for shared memory"); return ESPB_ERR_ARG; }
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(att_loc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { espb_set_error(cudaGetErrorString(e)); return ESPB_ERR_CUDA; }
  }
  espb::launch_pdl(att_loc_kernel, dim3(n), dim3(ATT_THREADS), smem, stream, enc_h, enc, enc_plane, lens, W, Tmax, A, E, dec_z, conv_w, chans,
                   filts, att_wt, gvec, gvec_b, anc, anc_ld, pos, step_ptr, ring, n, out, out_plane, out_ld, out2, out2_plane, out2_ld);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_drop_cand_i32(int* valid, int n, int PC, int j, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  if (j < 0 || j >= PC) { espb_set_error("drop_cand: need 0 <= j < PC"); return ESPB_ERR_ARG; }
  drop_cand_kernel<<<(n + 255) / 256, 256, 0, stream>>>(valid, n, PC, j);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

}  // extern "C"
