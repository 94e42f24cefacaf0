// Fused DefaultFrontend: framing (center=True, reflect pad) + periodic Hann + 512-point real FFT +
// power + sparse mel filterbank + clamp/log, one HBM read of the waveform and one write of the
// log-mel features, plus per-block column sums for UtteranceMVN (second tiny kernel subtracts).
//
// Reference: espnet2/layers/stft.py:75-120, espnet2/asr/frontend/default.py:82-117,
// espnet2/layers/log_mel.py:57-84, espnet2/layers/utterance_mvn.py:45-88.
#include <stdint.h>

#include "common.cuh"

namespace {

constexpr int NFFT = 512, NC = 256;  // NC: complex points of the packed FFT

struct MelSparse {          // filter m covers bins [start[m], start[m]+count[m]); weights packed at offset[m]
  const int* start; const int* count; const int* offset; const float* weight; int n_mels;
};

__device__ __forceinline__ int reflect_idx(int i, int L) {  // torch "reflect": no edge repeat
  if (i < 0) i = -i;
  if (i >= L) i = 2 * (L - 1) - i;
  return i;
}

// ---------------------------------------------------------------- register-resident FFT (v2)
// 16-point complex DFT in registers (forward, e^{-2 pi i nk/16}), radix 4 x 4: n = 4a + b, k = c + 4d.
struct c32 { float x, y; };
__device__ __forceinline__ c32 cmul(c32 a, c32 b) { return {a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }
__device__ __forceinline__ void dft4(c32 u0, c32 u1, c32 u2, c32 u3, c32& y0, c32& y1, c32& y2, c32& y3) {
  const c32 s02 = {u0.x + u2.x, u0.y + u2.y}, d02 = {u0.x - u2.x, u0.y - u2.y};
  const c32 s13 = {u1.x + u3.x, u1.y + u3.y}, d13 = {u1.x - u3.x, u1.y - u3.y};
  y0 = {s02.x + s13.x, s02.y + s13.y};
  y1 = {d02.x + d13.y, d02.y - d13.x};      // d02 - i d13
  y2 = {s02.x - s13.x, s02.y - s13.y};
  y3 = {d02.x - d13.y, d02.y + d13.x};      // d02 + i d13
}
__device__ __forceinline__ void dft16(c32 (&v)[16]) {
  // W16^m = (cos(2 pi m / 16), -sin(2 pi m / 16))
  constexpr float C1 = 0.92387953251128674f, S1 = 0.38268343236508977f, C2 = 0.70710678118654752f;
  c32 y[4][4];   // y[b][c]
#pragma unroll
  for (int b = 0; b < 4; ++b) dft4(v[b], v[4 + b], v[8 + b], v[12 + b], y[b][0], y[b][1], y[b][2], y[b][3]);
  // twiddles W16^{bc}: bc in {1,2,3,2,4,6,3,6,9}
  y[1][1] = cmul(y[1][1], {C1, -S1}); y[1][2] = cmul(y[1][2], {C2, -C2}); y[1][3] = cmul(y[1][3], {S1, -C1});
  y[2][1] = cmul(y[2][1], {C2, -C2}); y[2][2] = {y[2][2].y, -y[2][2].x};  y[2][3] = cmul(y[2][3], {-C2, -C2});
  y[3][1] = cmul(y[3][1], {S1, -C1}); y[3][2] = cmul(y[3][2], {-C2, -C2}); y[3][3] = cmul(y[3][3], {-C1, S1});
#pragma unroll
  for (int c = 0; c < 4; ++c) dft4(y[0][c], y[1][c], y[2][c], y[3][c], v[c], v[c + 4], v[c + 8], v[c + 12]);
}

// Half a warp transforms one frame, everything in registers: z[n] = x[2n] + i x[2n+1] (windowed), N = 256 = 16 x 16 four-step FFT
// (lane n2: 16-point DFT over n1 of z[16 n1 + n2]; twiddle W256^{n2 k1}; 16 x 16 transpose through a padded smem tile; lane k1: 16-point DFT
// over n2 -> Z[k1 + 16 k2]); real-FFT split with the mirror bin fetched by shuffle from lane 16 - k1; power -> smem; sparse mel + log.
// Generic hop length / window (any hop, window zero-padded to 512 taps by the host, stft.py:75-120); 32 frames per block, 4 warps.
constexpr int V2_WARPS = 4, V2_FPB = 32;
struct FrontV2Smem { int seg_floats; };
__global__ void __launch_bounds__(V2_WARPS * 32)
stft_logmel_v2_kernel(const float* __restrict__ wave, const long long* __restrict__ wave_lens, int Lmax, int hop, const float* __restrict__ window,
                      const float2* __restrict__ tw512, const float2* __restrict__ tw256t /* [k1][n2] = W256^{n2 k1} */, MelSparse mel, int mel_nnz,
                      float* __restrict__ out, int Tf_max, float* __restrict__ partial /* [B][nblk][n_mels] */) {
  extern __shared__ float smem[];
  const int seg_n = (V2_FPB - 1) * hop + NFFT;
  float* seg = smem;                                              // [seg_n] (rounded up to 4)
  float* win = seg + ((seg_n + 3) & ~3);                          // [512]
  float2* tw = reinterpret_cast<float2*>(win + NFFT);             // [256] W512^k
  float2* twt = tw + NC;                                          // [256] W256^{n2 k1} at [k1 * 16 + n2]
  float2* scr = twt + NC;                                         // [V2_WARPS][2][16 * 17] transpose tiles, reused as the power spectrum [260]
  float* melw = reinterpret_cast<float*>(scr + V2_WARPS * 2 * 16 * 17);   // [mel_nnz]
  int* mst = reinterpret_cast<int*>(melw + ((mel_nnz + 3) & ~3)); // start / count / offset [3][n_mels]
  float* colsum = reinterpret_cast<float*>(mst + 3 * mel.n_mels); // [V2_WARPS][2][n_mels]

  const int b = blockIdx.y, blk = blockIdx.x;
  const int L = (int)wave_lens[b];
  const int Tf = 1 + L / hop;
  const int f0 = blk * V2_FPB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, hl = lane & 15, half = lane >> 4;
  const float* w = wave + (long long)b * Lmax;
  const int nm = mel.n_mels;

  for (int i = threadIdx.x; i < NFFT; i += blockDim.x) win[i] = window[i];
  for (int i = threadIdx.x; i < NC; i += blockDim.x) { tw[i] = tw512[i]; twt[i] = tw256t[i]; }
  for (int i = threadIdx.x; i < mel_nnz; i += blockDim.x) melw[i] = mel.weight[i];
  for (int i = threadIdx.x; i < nm; i += blockDim.x) { mst[i] = mel.start[i]; mst[nm + i] = mel.count[i]; mst[2 * nm + i] = mel.offset[i]; }
  for (int i = threadIdx.x; i < V2_WARPS * 2 * nm; i += blockDim.x) colsum[i] = 0.f;
  const int s0 = f0 * hop - NFFT / 2;   // first (un-reflected) sample index of this block's segment
  if (L > 1) {
    const bool interior = s0 >= 0 && s0 + seg_n <= L && ((reinterpret_cast<uintptr_t>(w + s0) & 15) == 0);
    if (interior) {   // 128-bit loads: the block's samples are one contiguous, aligned run
      const float4* src = reinterpret_cast<const float4*>(w + s0);
      for (int i = threadIdx.x; i < (seg_n >> 2); i += blockDim.x) reinterpret_cast<float4*>(seg)[i] = __ldg(src + i);
      for (int i = (seg_n & ~3) + threadIdx.x; i < seg_n; i += blockDim.x) seg[i] = __ldg(w + s0 + i);
    } else {
      for (int i = threadIdx.x; i < seg_n; i += blockDim.x) {
        const int g = s0 + i;
        float v = 0.f;
        if (g < L + NFFT / 2 && g > -NFFT) v = __ldg(w + reflect_idx(g, L));
        seg[i] = v;
      }
    }
  } else {
    for (int i = threadIdx.x; i < seg_n; i += blockDim.x) seg[i] = 0.f;
  }
  __syncthreads();

  float2* T = scr + (warp * 2 + half) * (16 * 17);
  float* P = reinterpret_cast<float*>(T);
  float* csum = colsum + (warp * 2 + half) * nm;
  for (int it = 0; it < V2_FPB / (2 * V2_WARPS); ++it) {
    const int fl = it * 2 * V2_WARPS + warp * 2 + half;      // frame within the block
    const int f = f0 + fl;
    const bool live = f < Tf;                                // half-warp uniform; shuffles below stay warp-wide
    if (f < Tf_max && !live) {                               // padded frame of a shorter utterance: zeros (stft.py:117, log_mel.py:78-81)
      float* orow = out + ((long long)b * Tf_max + f) * nm;
      for (int m = hl; m < nm; m += 16) orow[m] = 0.f;
    }
    c32 v[16];
    {
      const float2* x2 = reinterpret_cast<const float2*>(seg + fl * hop);    // hop even -> 8-byte aligned; odd hops take the scalar path
      const float2* w2 = reinterpret_cast<const float2*>(win);
      const bool al = ((fl * hop) & 1) == 0;
#pragma unroll
      for (int n1 = 0; n1 < 16; ++n1) {
        const int n = 16 * n1 + hl;
        float2 xv;
        if (al) xv = x2[n]; else { xv.x = seg[fl * hop + 2 * n]; xv.y = seg[fl * hop + 2 * n + 1]; }
        const float2 wv = w2[n];
        v[n1] = {live ? xv.x * wv.x : 0.f, live ? xv.y * wv.y : 0.f};
      }
    }
    dft16(v);                                                // v[k1] = sum_n1 z[16 n1 + n2] W16^{n1 k1}
#pragma unroll
    for (int k1 = 1; k1 < 16; ++k1) { const float2 t = twt[k1 * 16 + hl]; v[k1] = cmul(v[k1], {t.x, t.y}); }
    __syncwarp();
#pragma unroll
    for (int k1 = 0; k1 < 16; ++k1) T[hl * 17 + k1] = make_float2(v[k1].x, v[k1].y);
    __syncwarp();
#pragma unroll
    for (int n2 = 0; n2 < 16; ++n2) { const float2 t = T[n2 * 17 + hl]; v[n2] = {t.x, t.y}; }
    dft16(v);                                                // v[k2] = Z[hl + 16 k2]
    __syncwarp();                                            // tile reads done: it becomes the power spectrum
    // real split: X[k] = (Z[k] + conj Z[N-k]) / 2 - i/2 w^k (Z[k] - conj Z[N-k]),  N - k = (16 - k1) + 16 (15 - k2)
    const int src = ((16 - hl) & 15) + 16 * half;
#pragma unroll
    for (int k2 = 0; k2 < 16; ++k2) {
      float znx = __shfl_sync(0xffffffffu, v[15 - k2].x, src), zny = __shfl_sync(0xffffffffu, v[15 - k2].y, src);
      if (hl == 0) { znx = v[(16 - k2) & 15].x; zny = v[(16 - k2) & 15].y; }
      const c32 zk = v[k2];
      const c32 e = {0.5f * (zk.x + znx), 0.5f * (zk.y - zny)}, o = {0.5f * (zk.x - znx), 0.5f * (zk.y + zny)};
      const float2 t = tw[hl + 16 * k2];
      const float tox = t.x * o.x - t.y * o.y, toy = t.x * o.y + t.y * o.x;
      const float re = e.x + toy, im = e.y - tox;
      P[hl + 16 * k2] = re * re + im * im;
    }
    if (hl == 0) { const float d = v[0].x - v[0].y; P[NC] = d * d; }
    __syncwarp();
    if (live) {
      float* orow = out + ((long long)b * Tf_max + f) * nm;
      for (int m = hl; m < nm; m += 16) {
        const int st0 = mst[m], cnt = mst[nm + m];
        const float* wm = melw + mst[2 * nm + m];
        float acc = 0.f;
        for (int i = 0; i < cnt; ++i) acc = fmaf(P[st0 + i], wm[i], acc);
        const float lv = logf(fmaxf(acc, 1e-10f));
        orow[m] = lv;
        csum[m] += lv;
      }
    }
    __syncwarp();
  }
  __syncthreads();
  if (partial) {
    for (int m = threadIdx.x; m < nm; m += blockDim.x) {
      float sacc = 0.f;
#pragma unroll
      for (int q = 0; q < V2_WARPS * 2; ++q) sacc += colsum[q * nm + m];
      partial[((long long)b * gridDim.x + blk) * nm + m] = sacc;
    }
  }
}

// UtteranceMVN (norm_means only): x[b,t,:] -= sum_t x[b,t,:] / Tf_b for valid frames; padded frames stay 0.
__global__ void utt_mvn_kernel(float* __restrict__ feats, const long long* __restrict__ wave_lens, int Tf_max, int n_mels, int hop,
                               const float* __restrict__ partial, int nblk) {
  __shared__ float mean[128];
  const int b = blockIdx.y;
  const int Tf = 1 + (int)wave_lens[b] / hop;
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    float s = 0.f;
    for (int i = 0; i < nblk; ++i) s += partial[((long long)b * nblk + i) * n_mels + m];
    mean[m] = s / (float)Tf;
  }
  __syncthreads();
  const int t0 = blockIdx.x * 32;
  for (int i = threadIdx.x; i < 32 * n_mels; i += blockDim.x) {
    int t = t0 + i / n_mels, m = i % n_mels;
    if (t < Tf) feats[((long long)b * Tf_max + t) * n_mels + m] -= mean[m];
  }
}

// Column sums over valid frames for features that did not come from stft_logmel_v2_kernel (standalone normalize).
__global__ void feat_colsum_kernel(const float* __restrict__ feats, const long long* __restrict__ feat_lens, int Tf_max, int n_mels,
                                   float* __restrict__ partial, int nblk) {
  const int b = blockIdx.y, blk = blockIdx.x;
  const int Tf = (int)feat_lens[b];
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    float s = 0.f;
    for (int t = blk * 32; t < min(Tf, blk * 32 + 32); ++t) s += feats[((long long)b * Tf_max + t) * n_mels + m];
    partial[((long long)b * nblk + blk) * n_mels + m] = s;
  }
}

__global__ void utt_mvn_feat_kernel(float* __restrict__ feats, const long long* __restrict__ feat_lens, int Tf_max, int n_mels,
                                    const float* __restrict__ partial, int nblk) {
  __shared__ float mean[128];
  const int b = blockIdx.y;
  const int Tf = (int)feat_lens[b];
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    float s = 0.f;
    for (int i = 0; i < nblk; ++i) s += partial[((long long)b * nblk + i) * n_mels + m];
    mean[m] = s / (float)Tf;
  }
  __syncthreads();
  const int t0 = blockIdx.x * 32;
  for (int i = threadIdx.x; i < 32 * n_mels; i += blockDim.x) {
    int t = t0 + i / n_mels, m = i % n_mels;
    if (t < Tf) feats[((long long)b * Tf_max + t) * n_mels + m] -= mean[m];
  }
}

// GlobalMVN.forward (espnet2/layers/global_mvn.py:74-103): (x - mean) on valid frames, padded frames 0, then / std.
__global__ void global_mvn_kernel(float* __restrict__ feats, const long long* __restrict__ feat_lens, int Tmax, int D, const float* __restrict__ mean,
                                  const float* __restrict__ stdv, int norm_means, int norm_vars) {
  const int b = blockIdx.y;
  const long long n = (long long)Tmax * D;
  const int Tf = (int)feat_lens[b];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / D), d = (int)(i % D);
    float v = feats[(long long)b * n + i];
    if (norm_means) v -= mean[d];
    if (t >= Tf) v = 0.f;
    if (norm_vars) v /= stdv[d];
    feats[(long long)b * n + i] = v;
  }
}

}  // namespace

extern "C" {

int espb_frontend_blocks(int Tf_max) { return (Tf_max + V2_FPB - 1) / V2_FPB; }

int espb_stft_logmel_f32(const float* wave, const long long* wave_lens, int B, int Lmax, int hop, const float* window,
                         const float* tw512, const float* tw256t, const int* mel_start, const int* mel_count, const int* mel_offset,
                         const float* mel_weight, int mel_nnz, int n_mels, float* out, int Tf_max, float* partial, cudaStream_t stream) {
  if (B <= 0 || Lmax <= 0 || n_mels <= 0 || n_mels > 128 || hop <= 0 || hop > 1024 || mel_nnz < 0 || mel_nnz > 4096) {
    espb_set_error("stft_logmel: bad shape (n_mels <= 128, 0 < hop <= 1024, mel non-zeros <= 4096)"); return ESPB_ERR_ARG;
  }
  MelSparse mel{mel_start, mel_count, mel_offset, mel_weight, n_mels};
  dim3 grid(espb_frontend_blocks(Tf_max), B);
  const int seg_n = (V2_FPB - 1) * hop + NFFT;
  const size_t smem = ((size_t)((seg_n + 3) & ~3) + NFFT + 2 * NC * 2 + (size_t)V2_WARPS * 2 * 16 * 17 * 2 + ((mel_nnz + 3) & ~3) + 3 * n_mels +
                       (size_t)V2_WARPS * 2 * n_mels) * sizeof(float);
  if (smem > 200 * 1024) { espb_set_error("stft_logmel: hop too large for shared memory"); return ESPB_ERR_ARG; }
  static size_t attr_smem = 0;
  if (smem > 48 * 1024 && smem > attr_smem) {
    if (cudaFuncSetAttribute(stft_logmel_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)) != cudaSuccess) {
      espb_set_error("stft_logmel: cannot raise dynamic shared memory"); return ESPB_ERR_CUDA;
    }
    attr_smem = 200 * 1024;
  }
  stft_logmel_v2_kernel<<<grid, V2_WARPS * 32, smem, stream>>>(wave, wave_lens, Lmax, hop, window, reinterpret_cast<const float2*>(tw512),
                                                              reinterpret_cast<const float2*>(tw256t), mel, mel_nnz, out, Tf_max, partial);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_utt_mvn_from_partial_f32(float* feats, const long long* wave_lens, int B, int Tf_max, int n_mels, int hop, const float* partial,
                                  cudaStream_t stream) {
  if (n_mels > 128) { espb_set_error("utt_mvn: n_mels > 128"); return ESPB_ERR_ARG; }
  dim3 grid((Tf_max + 31) / 32, B);
  utt_mvn_kernel<<<grid, 256, 0, stream>>>(feats, wave_lens, Tf_max, n_mels, hop, partial, espb_frontend_blocks(Tf_max));
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_utt_mvn_f32(float* feats, const long long* feat_lens, int B, int Tf_max, int n_mels, float* partial_ws, cudaStream_t stream) {
  if (n_mels > 128) { espb_set_error("utt_mvn: n_mels > 128"); return ESPB_ERR_ARG; }
  const int nblk = (Tf_max + 31) / 32;
  dim3 grid(nblk, B);
  feat_colsum_kernel<<<grid, 128, 0, stream>>>(feats, feat_lens, Tf_max, n_mels, partial_ws, nblk);
  utt_mvn_feat_kernel<<<grid, 256, 0, stream>>>(feats, feat_lens, Tf_max, n_mels, partial_ws, nblk);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_global_mvn_f32(float* feats, const long long* feat_lens, int B, int Tmax, int D, const float* mean, const float* stdv, int norm_means,
                        int norm_vars, cudaStream_t stream) {
  dim3 grid(64, B);
  global_mvn_kernel<<<grid, 256, 0, stream>>>(feats, feat_lens, Tmax, D, mean, stdv, norm_means, norm_vars);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

}  // extern "C"
