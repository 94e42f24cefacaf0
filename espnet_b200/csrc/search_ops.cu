// Device-resident joint CTC/attention beam search, batched over utterances (U) x beam slots (W).
// Slot s = u*W + w.  All hypotheses of a step have the same length, so the step index is a launch
// argument; per-slot state (scores, CTC forward variables, ancestor table of the self-attention
// cache) lives in HBM and is double-buffered across steps.
//
// Reference semantics: espnet2/legacy/nets/batch_beam_search.py:253-357,359-423 (search, post_process),
// beam_search.py:385-498 (loop, maxlen/minlen), e2e_asr_common.py:14-44 (end_detect),
// ctc_prefix_score.py:71-191 + scorers/ctc.py:40-63,101-126 (CTC prefix scorer),
// asr/decoder/transformer_decoder.py:191-311 + transformer/decoder_layer.py:73-179 (decoder step).
#include <stdlib.h>

#include "common.cuh"

namespace {

constexpr float LOGZERO = -10000000000.0f;  // ctc_prefix_score.py:34
using espb::logaddexp;

__device__ __forceinline__ void store_split(float* p, long long plane, float v) {
  float h = espb::tf32_hi(v);
  p[0] = h;
  p[plane] = espb::tf32_lo(v, h);
}

// ---------------------------------------------------------------- decoder input: embed(last token)*sqrt(D) + PE[pos]
__global__ void dec_embed_kernel(const int* __restrict__ last_tok, const float* __restrict__ emb, const float* __restrict__ pe, int pos,
                                 const int* __restrict__ step_ptr, int D, float scale, float* __restrict__ x) {
  espb::pdl_trigger();
  espb::pdl_wait();
  if (step_ptr) pos += *step_ptr;
  const int s = blockIdx.x;
  const float* e = emb + (long long)last_tok[s] * D;
  const float* p = pe + (long long)pos * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) x[(long long)s * D + c] = e[c] * scale + p[c];
}

// ---------------------------------------------------------------- self-attention of the newest token over the prefix
// qkv [n][3D] (this step's q,k,v, bias added). K/V of earlier positions j < pos live in kc/vc [Lmax][n][D] at slot anc[s][j].
// Writes this step's k,v into kc/vc[pos][s] and ctx (split) [n][D].  One warp per (slot, head); lanes split d_k (<= 128) so
// that every K/V row is one coalesced read; 4 positions are in flight per iteration.
__global__ void __launch_bounds__(128) dec_self_attn_kernel(const float* __restrict__ qkv, float* __restrict__ kc, float* __restrict__ vc,
                                                            const int* __restrict__ anc, int anc_ld, int n, int D, int H, int pos,
                                                            const int* __restrict__ step_ptr, int sc_ld, float* __restrict__ ctx,
                                                            long long ctx_plane) {
  extern __shared__ float sm[];  // per warp: sc_ld >= pos+1 scores
  espb::pdl_trigger();
  espb::pdl_wait();
  if (step_ptr) pos += *step_ptr;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wid = blockIdx.x * (blockDim.x >> 5) + warp;
  if (wid >= n * H) return;
  const int s = wid / H, h = wid % H, dk = D / H;
  float* sc = sm + warp * sc_ld;
  const float* q = qkv + (long long)s * 3 * D + h * dk;
  float qr[4], kn[4], vn[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int d = lane + 32 * i;
    qr[i] = (d < dk) ? q[d] : 0.f;
    kn[i] = (d < dk) ? q[D + d] : 0.f;
    vn[i] = (d < dk) ? q[2 * D + d] : 0.f;
    if (d < dk) {   // append this step's k, v to the cache
      kc[((long long)pos * n + s) * D + h * dk + d] = kn[i];
      vc[((long long)pos * n + s) * D + h * dk + d] = vn[i];
    }
  }
  const float rs = sqrtf((float)dk);
  const int* an = anc + (long long)s * anc_ld;
  for (int j0 = 0; j0 <= pos; j0 += 8) {
    float part[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int j = j0 + u;
      float a = 0.f;
      if (j < pos) {
        const float* kj = kc + ((long long)j * n + an[j]) * D + h * dk;
#pragma unroll
        for (int i = 0; i < 4; ++i) { const int d = lane + 32 * i; if (d < dk) a = fmaf(qr[i], kj[d], a); }
      } else if (j == pos) {
#pragma unroll
        for (int i = 0; i < 4; ++i) a = fmaf(qr[i], kn[i], a);
      }
      part[u] = a;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float a = espb::warp_sum(part[u]);
      if (lane == 0 && j0 + u <= pos) sc[j0 + u] = a / rs;
    }
  }
  __syncwarp();
  float mx = -INFINITY;
  for (int j = lane; j <= pos; j += 32) mx = fmaxf(mx, sc[j]);
  mx = espb::warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j <= pos; j += 32) { float e = expf(sc[j] - mx); sc[j] = e; sum += e; }
  sum = espb::warp_sum(sum);
  __syncwarp();
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < pos; ++j) {
    const float pj = sc[j] / sum;
    const float* vj = vc + ((long long)j * n + an[j]) * D + h * dk;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const int d = lane + 32 * i; if (d < dk) acc[i] = fmaf(pj, vj[d], acc[i]); }
  }
  {
    const float pj = sc[pos] / sum;
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i] = fmaf(pj, vn[i], acc[i]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int d = lane + 32 * i;
    if (d < dk) store_split(ctx + (long long)s * D + h * dk + d, ctx_plane, acc[i]);
  }
}

// d_k = 64 instance: a half-warp covers one 256-byte K / V row with 128-bit loads, so every load instruction fetches two prefix
// positions; ancestor slots of 32 positions are read with one coalesced load and broadcast by shuffle (no dependent
// index -> row load chain); dot products reduce over 16 lanes.
__global__ void __launch_bounds__(128) dec_self_attn64_kernel(const float* __restrict__ qkv, float* __restrict__ kc, float* __restrict__ vc,
                                                              const int* __restrict__ anc, int anc_ld, int n, int D, int H, int pos,
                                                              const int* __restrict__ step_ptr, int sc_ld, float* __restrict__ ctx,
                                                              long long ctx_plane) {
  extern __shared__ float sm[];  // per warp: sc_ld >= pos+1 scores
  espb::pdl_trigger();
  espb::pdl_wait();
  if (step_ptr) pos += *step_ptr;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wid = blockIdx.x * (blockDim.x >> 5) + warp;
  if (wid >= n * H) return;
  const int s = wid / H, h = wid % H;
  const int half = lane >> 4, l16 = lane & 15;
  float* sc = sm + warp * sc_ld;
  const float* q = qkv + (long long)s * 3 * D + h * 64 + 4 * l16;
  const float4 q4 = *reinterpret_cast<const float4*>(q);
  const float4 kn = *reinterpret_cast<const float4*>(q + D);
  const float4 vn = *reinterpret_cast<const float4*>(q + 2 * D);
  if (half == 0) {   // append this step's k, v to the cache
    *reinterpret_cast<float4*>(kc + ((long long)pos * n + s) * D + h * 64 + 4 * l16) = kn;
    *reinterpret_cast<float4*>(vc + ((long long)pos * n + s) * D + h * 64 + 4 * l16) = vn;
  }
  const int* an = anc + (long long)s * anc_ld;
  const long long hoff = (long long)h * 64 + 4 * l16;
  for (int j0 = 0; j0 <= pos; j0 += 32) {
    const int my_a = (j0 + lane < pos) ? an[j0 + lane] : 0;
#pragma unroll
    for (int it0 = 0; it0 < 16; it0 += 8) {
      if (j0 + 2 * it0 > pos) break;          // warp-uniform
      float part[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int jj = 2 * (it0 + u) + half, j = j0 + jj;
        const int aj = __shfl_sync(0xffffffffu, my_a, jj);
        float a = 0.f;
        if (j < pos) {
          const float4 k4 = *reinterpret_cast<const float4*>(kc + ((long long)j * n + aj) * D + hoff);
          a = fmaf(q4.x, k4.x, fmaf(q4.y, k4.y, fmaf(q4.z, k4.z, q4.w * k4.w)));
        } else if (j == pos) {
          a = fmaf(q4.x, kn.x, fmaf(q4.y, kn.y, fmaf(q4.z, kn.z, q4.w * kn.w)));
        }
        part[u] = a;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        float a = part[u];
        a += __shfl_xor_sync(0xffffffffu, a, 8); a += __shfl_xor_sync(0xffffffffu, a, 4);
        a += __shfl_xor_sync(0xffffffffu, a, 2); a += __shfl_xor_sync(0xffffffffu, a, 1);
        const int j = j0 + 2 * (it0 + u) + half;
        if (l16 == 0 && j <= pos) sc[j] = a / 8.0f;
      }
    }
  }
  __syncwarp();
  float mx = -INFINITY;
  for (int j = lane; j <= pos; j += 32) mx = fmaxf(mx, sc[j]);
  mx = espb::warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j <= pos; j += 32) { float e = expf(sc[j] - mx); sc[j] = e; sum += e; }
  sum = espb::warp_sum(sum);
  __syncwarp();
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j0 = 0; j0 < pos; j0 += 32) {
    const int my_a = (j0 + lane < pos) ? an[j0 + lane] : 0;
#pragma unroll 8
    for (int it = 0; it < 16; ++it) {
      const int jj = 2 * it + half, j = j0 + jj;
      if (j0 + 2 * it >= pos) break;          // warp-uniform
      const int aj = __shfl_sync(0xffffffffu, my_a, jj);
      if (j < pos) {
        const float pj = sc[j] / sum;
        const float4 v4 = *reinterpret_cast<const float4*>(vc + ((long long)j * n + aj) * D + hoff);
        acc.x = fmaf(pj, v4.x, acc.x); acc.y = fmaf(pj, v4.y, acc.y); acc.z = fmaf(pj, v4.z, acc.z); acc.w = fmaf(pj, v4.w, acc.w);
      }
    }
  }
  acc.x += __shfl_xor_sync(0xffffffffu, acc.x, 16); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, 16);
  acc.z += __shfl_xor_sync(0xffffffffu, acc.z, 16); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, 16);
  if (half == 0) {
    const float pj = sc[pos] / sum;
    acc.x = fmaf(pj, vn.x, acc.x); acc.y = fmaf(pj, vn.y, acc.y); acc.z = fmaf(pj, vn.z, acc.z); acc.w = fmaf(pj, vn.w, acc.w);
    float4 hi, lo;
    hi.x = espb::tf32_hi(acc.x); hi.y = espb::tf32_hi(acc.y); hi.z = espb::tf32_hi(acc.z); hi.w = espb::tf32_hi(acc.w);
    lo.x = espb::tf32_lo(acc.x, hi.x); lo.y = espb::tf32_lo(acc.y, hi.y); lo.z = espb::tf32_lo(acc.z, hi.z); lo.w = espb::tf32_lo(acc.w, hi.w);
    float* o = ctx + (long long)s * D + hoff;
    *reinterpret_cast<float4*>(o) = hi;
    *reinterpret_cast<float4*>(o + ctx_plane) = lo;
  }
}

// ---------------------------------------------------------------- cross-attention of W queries per utterance over the encoder memory
// q [n][D]; memory K / V blocks are contiguous per (utterance, head): kmem/vmem + ((u*H + h)*Tmax + t)*dk + d  (written once per
// utterance by the K/V projection GEMMs and shared by the whole beam).  One block per (utterance, head): the K and V blocks are
// streamed exactly once with coalesced 128-bit loads (LPR lanes per row, several rows per warp instruction, UN instructions in flight).
// WC / DKC: compile-time beam size / head dim (0 = run-time values): the specialised instances have no predicates in the inner loops.
template <int UN, int WC, int DKC>
__global__ void __launch_bounds__(256, 3) dec_src_attn_kernel(const float* __restrict__ q, const float* __restrict__ kmem, const float* __restrict__ vmem,
                                                           int Tmax, const int* __restrict__ lens, int W_rt, int D, int H, int lpr_rt /* pow2 >= dk/4 */,
                                                           float* __restrict__ ctx, long long ctx_plane, int w0, int Wall) {
  extern __shared__ float sm[];  // q [W][dk] | scores [W][Tmax] (reused for the cross-warp PV reduction) | K tile [128][dk+4]
  espb::pdl_trigger();
  espb::pdl_wait();
  constexpr bool CT = (WC > 0);
  constexpr int JMAX = CT ? (WC + 1) / 2 : 8;          // beam slots per half block
  constexpr bool FULL = CT && (WC % 2 == 0);           // both halves own exactly JMAX slots
  const int W = CT ? WC : W_rt;
  const int dk = (DKC > 0) ? DKC : D / H;
  const int lpr = (DKC == 64) ? 16 : lpr_rt;
  const int u = blockIdx.x / H, h = blockIdx.x % H;
  const int T = lens[u];
  float* qs = sm;
  float* sc = qs + W * dk;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  for (int i = threadIdx.x; i < W * dk; i += blockDim.x) qs[i] = q[((long long)(u * Wall + w0 + i / dk)) * D + h * dk + (i % dk)];   // slots w0 .. w0+W-1 of the Wall beam slots
  __syncthreads();
  const int rpw = 32 / lpr;                 // rows per warp instruction
  const int rsub = lane / lpr, c4 = lane % lpr;   // row within the group, float4 column
  const bool col_ok = c4 * 4 < dk;
  const float rs = sqrtf((float)dk);
  const float4* kb = reinterpret_cast<const float4*>(kmem + ((long long)(u * H + h) * Tmax) * dk);
  const float4* vb = reinterpret_cast<const float4*>(vmem + ((long long)(u * H + h) * Tmax) * dk);
  const int dk4 = dk / 4;
  // ---- scores[w][t] = q_w . k_t / sqrt(dk): K tiles of 128 rows are staged in smem with coalesced 128-bit loads, then each thread
  // owns one row (held in registers) and half of the beam slots: in-lane dot products, no shuffles.
  {
    float* kt = sc + (((long long)W * Tmax + 3) & ~3LL);   // [128][dk + 4], 16-byte aligned
    const int kst = dk + 4;
    const int r = threadIdx.x & 127, half = threadIdx.x >> 7;
    const int w_lo = half * ((W + 1) / 2), w_hi = min(W, w_lo + (W + 1) / 2);
    for (int tb = 0; tb < T; tb += 128) {
      const int rows = min(128, T - tb);
      for (int i = threadIdx.x; i < rows * dk4; i += blockDim.x) {
        const int rr = i / dk4, cc = i % dk4;
        *reinterpret_cast<float4*>(kt + rr * kst + cc * 4) = __ldg(kb + (long long)(tb + rr) * dk4 + cc);
      }
      __syncthreads();
      if (r < rows) {
        float a[JMAX];
#pragma unroll
        for (int j = 0; j < JMAX; ++j) a[j] = 0.f;
        for (int d0 = 0; d0 < dk; d0 += 4) {
          const float4 k4 = *reinterpret_cast<const float4*>(kt + r * kst + d0);
#pragma unroll
          for (int j = 0; j < JMAX; ++j) {
            const int w = w_lo + j;
            if (FULL || w < w_hi) {
              const float4 q4 = *reinterpret_cast<const float4*>(qs + w * dk + d0);
              a[j] = fmaf(q4.x, k4.x, a[j]); a[j] = fmaf(q4.y, k4.y, a[j]); a[j] = fmaf(q4.z, k4.z, a[j]); a[j] = fmaf(q4.w, k4.w, a[j]);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < JMAX; ++j) if (FULL || w_lo + j < w_hi) sc[(w_lo + j) * Tmax + tb + r] = a[j] / rs;
      }
      __syncthreads();
    }
  }
  __syncthreads();
  // ---- softmax over t per slot (no memory mask: batch_score passes none, transformer_decoder.py:294-303)
  for (int w = warp; w < W; w += nwarp) {
    float* r = sc + w * Tmax;
    float mx = -INFINITY;
    for (int t = lane; t < T; t += 32) mx = fmaxf(mx, r[t]);
    mx = espb::warp_max(mx);
    float sum = 0.f;
    for (int t = lane; t < T; t += 32) { float e = expf(r[t] - mx); r[t] = e; sum += e; }
    sum = espb::warp_sum(sum);
    for (int t = lane; t < T; t += 32) r[t] = r[t] / sum;
  }
  __syncthreads();
  // ---- ctx[w][d] = sum_t p[w][t] * v[t][d]: the two halves of the block own the two halves of the beam slots (8 accumulators per
  // lane); each half streams V with coalesced 128-bit loads, UN row groups in flight per warp.
  const int hw = nwarp >> 1, hf = warp / hw, wh = warp % hw;
  const int w_lo = hf * ((W + 1) / 2), w_hi = min(W, w_lo + (W + 1) / 2);
  float4 acc[JMAX];
#pragma unroll
  for (int j = 0; j < JMAX; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int t0 = wh * rpw * UN; t0 < T; t0 += hw * rpw * UN) {
    float4 vv[UN];
#pragma unroll
    for (int uu = 0; uu < UN; ++uu) {
      const int t = t0 + uu * rpw + rsub;
      vv[uu] = (t < T && col_ok) ? __ldg(vb + (long long)t * dk4 + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int uu = 0; uu < UN; ++uu) {
      const int t = min(t0 + uu * rpw + rsub, T - 1);   // rows beyond T carry v = 0
#pragma unroll
      for (int j = 0; j < JMAX; ++j) {
        if (FULL || w_lo + j < w_hi) {
          const float pw = sc[(w_lo + j) * Tmax + t];
          acc[j].x = fmaf(pw, vv[uu].x, acc[j].x); acc[j].y = fmaf(pw, vv[uu].y, acc[j].y);
          acc[j].z = fmaf(pw, vv[uu].z, acc[j].z); acc[j].w = fmaf(pw, vv[uu].w, acc[j].w);
        }
      }
    }
  }
  // reduce over the rpw row groups of the warp (lanes with equal c4), then across the warps of the half through smem
#pragma unroll
  for (int j = 0; j < JMAX; ++j) {
    if (FULL || w_lo + j < w_hi) {
      for (int o = lpr; o < 32; o <<= 1) {
        acc[j].x += __shfl_xor_sync(0xffffffffu, acc[j].x, o); acc[j].y += __shfl_xor_sync(0xffffffffu, acc[j].y, o);
        acc[j].z += __shfl_xor_sync(0xffffffffu, acc[j].z, o); acc[j].w += __shfl_xor_sync(0xffffffffu, acc[j].w, o);
      }
    }
  }
  __syncthreads();   // probabilities are dead: reuse the score area as red[hw][W][dk]
  float* red = sc;
  if (rsub == 0 && col_ok) {
#pragma unroll
    for (int j = 0; j < JMAX; ++j)
      if (FULL || w_lo + j < w_hi) *reinterpret_cast<float4*>(red + ((long long)wh * W + w_lo + j) * dk + c4 * 4) = acc[j];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < W * dk; i += blockDim.x) {
    float a = 0.f;
    for (int g = 0; g < hw; ++g) a += red[(long long)g * W * dk + i];
    store_split(ctx + ((long long)(u * Wall + w0 + i / dk)) * D + h * dk + (i % dk), ctx_plane, a);
  }
}

// ---------------------------------------------------------------- cross-attention on the tensor cores (d_k = 64, beam <= 16)
// Same contract as dec_src_attn_kernel.  Scores S[t][slot] = K_tile[t][:] . Q[slot][:] and the context O[slot][d] = sum_t P[slot][t] V[t][d] are
// m16n8k8 TF32 mma.sync products with the 3xTF32 error compensation (operands split into hi/lo in registers), fed from smem-staged K / V
// tiles; this removes ~4/5 of the FFMA/LDS instructions that bound the CUDA-core version (ncu: 99 M warp instructions, 46 % issue-active).
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi)) & 0xFFFFE000u;
}
__device__ __forceinline__ void mma_m16n8k8_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma3_tf32(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const uint32_t (&bh)[2], const uint32_t (&bl)[2]) {
  mma_m16n8k8_tf32(c, al, bh);
  mma_m16n8k8_tf32(c, ah, bl);
  mma_m16n8k8_tf32(c, ah, bh);
}

__device__ __forceinline__ void cp_async16_zfill(float* smem_dst, const void* gsrc, int src_bytes) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// The K tiles and then the V tiles of one (utterance, head) stream through an S-deep cp.async ring of 64-frame tiles (one
// __syncthreads per tile; S-1 tiles in flight per block, two blocks per SM), so the HBM read of the encoder memory -- the
// algorithmic cost of this kernel -- is never stalled behind the mma phases; the softmax runs while the first V tiles land.
template <int S>
__global__ void __launch_bounds__(256, 2) dec_src_attn_mma_kernel(const float* __restrict__ q, const float* __restrict__ kmem, const float* __restrict__ vmem,
                                                                  int Tmax, const int* __restrict__ lens, int W, int D, int H,
                                                                  float* __restrict__ ctx, long long ctx_plane, int w0, int Wall) {
  constexpr int DK = 64, QST = 68, KST = 68, VST = 72, TR = 64, TILE_F = TR * VST;
  extern __shared__ float sm[];  // q [16][68] | scores [W][Tmax] (pad 4) | ring [S][64][72] (reused for the cross-warp reduction)
  espb::pdl_trigger();
  espb::pdl_wait();
  const int u = blockIdx.x / H, h = blockIdx.x % H;
  const int T = lens[u];
  float* qs = sm;
  float* sc = qs + 16 * QST;
  float* ring = sc + (((long long)W * Tmax + 3) & ~3LL);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const float4* kb = reinterpret_cast<const float4*>(kmem + ((long long)(u * H + h) * Tmax) * DK);
  const float4* vb = reinterpret_cast<const float4*>(vmem + ((long long)(u * H + h) * Tmax) * DK);
  const int nt = (T + TR - 1) / TR, NT = 2 * nt;
  auto issue = [&](int i) {
    if (i < NT) {
      const bool isk = i < nt;
      const int tb = (isk ? i : i - nt) * TR;
      const float4* src = isk ? kb : vb;
      const int st = isk ? KST : VST;
      float* dst = ring + (i % S) * TILE_F;
#pragma unroll
      for (int j = threadIdx.x; j < TR * 16; j += 256) {
        const int rr = j >> 4, cc = j & 15;
        const bool ok = tb + rr < T;      // frames past the utterance are zero-filled (src-size 0)
        cp_async16_zfill(dst + rr * st + cc * 4, src + (ok ? (long long)(tb + rr) * 16 + cc : 0), ok ? 16 : 0);
      }
    }
    cp_async_commit();                    // one (possibly empty) group per tile index keeps the wait_group arithmetic uniform
  };
#pragma unroll
  for (int i = 0; i < S - 1; ++i) issue(i);
  for (int i = threadIdx.x; i < 16 * DK; i += blockDim.x) {
    const int w = i / DK, d = i % DK;
    qs[w * QST + d] = (w < W) ? q[((long long)(u * Wall + w0 + w)) * D + h * DK + d] : 0.f;
  }
  const float rs = 8.0f;   // sqrt(d_k)
  const int sa = min(g, W - 1), sb = min(g + 8, W - 1);
  __syncthreads();         // qs is complete

  // ================================================================= K phase: S[slot][t] = Q[slot][:] . K[t][:]
  // A = Q (16 slot rows x 8 d per k-step, the same for every tile: split once into registers), B = K^T (8 d x 8 frames): warp w owns
  // frames 8w..8w+7 of each 64-frame tile, so every K element is read from smem and split exactly once (the earlier layout -- A = K rows,
  // B = Q^T -- split every K element in two warps and re-split Q for every tile: 3x the instructions of this loop; the kernel is
  // issue-bound, not HBM-bound: ncu r01 30 % tensor pipe, 2.9 TB/s).
  {
    uint32_t qh[8][4], ql[8][4];
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      split_tf32(qs[g * QST + ks * 8 + t4], qh[ks][0], ql[ks][0]);
      split_tf32(qs[(g + 8) * QST + ks * 8 + t4], qh[ks][1], ql[ks][1]);
      split_tf32(qs[g * QST + ks * 8 + t4 + 4], qh[ks][2], ql[ks][2]);
      split_tf32(qs[(g + 8) * QST + ks * 8 + t4 + 4], qh[ks][3], ql[ks][3]);
    }
    for (int i = 0; i < nt; ++i) {
      cp_async_wait<S - 2>();               // this thread's copies of tile i have landed ...
      __syncthreads();                      // ... and everyone's; all warps are done with tile i-1, whose slot is refilled next
      issue(i + S - 1);
      const float* tile = ring + (i % S) * TILE_F;
      const int tb = i * TR, rows = min(TR, T - tb);
      const int f0 = warp * 8;
      if (f0 < rows) {
        // one accumulator per product term: three independent 8-deep mma chains instead of one 24-deep chain
        float c[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f}, c2[4] = {0.f, 0.f, 0.f, 0.f};
        const float* kr = tile + (f0 + g) * KST + t4;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
          uint32_t bh[2], bl[2];
          split_tf32(kr[ks * 8], bh[0], bl[0]);
          split_tf32(kr[ks * 8 + 4], bh[1], bl[1]);
          mma_m16n8k8_tf32(c1, ql[ks], bh);
          mma_m16n8k8_tf32(c2, qh[ks], bl);
          mma_m16n8k8_tf32(c, qh[ks], bh);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) c[e] += c1[e] + c2[e];   // small terms combined first
        const int fa = tb + f0 + 2 * t4;                      // C fragment: rows (slots) g, g+8; columns (frames) 2*t4, 2*t4+1
        if (g < W) { if (fa < T) sc[g * Tmax + fa] = c[0] / rs; if (fa + 1 < T) sc[g * Tmax + fa + 1] = c[1] / rs; }
        if (g + 8 < W) { if (fa < T) sc[(g + 8) * Tmax + fa] = c[2] / rs; if (fa + 1 < T) sc[(g + 8) * Tmax + fa + 1] = c[3] / rs; }
      }
    }
  }

  // ================================================================= V phase: O[slot][d] = sum_t P[slot][t] V[t][d]
  float acc[8][4];
#pragma unroll
  for (int n8 = 0; n8 < 8; ++n8) { acc[n8][0] = 0.f; acc[n8][1] = 0.f; acc[n8][2] = 0.f; acc[n8][3] = 0.f; }
  for (int i = nt; i < NT; ++i) {
    cp_async_wait<S - 2>();
    __syncthreads();
    issue(i + S - 1);
    if (i == nt) {
      // ---- softmax over t per slot (no memory mask: batch_score passes none, transformer_decoder.py:294-303); the first V tiles land meanwhile
      for (int w = warp; w < W; w += 8) {
        float* r = sc + w * Tmax;
        float mx = -INFINITY;
        for (int t = lane; t < T; t += 32) mx = fmaxf(mx, r[t]);
        mx = espb::warp_max(mx);
        float sum = 0.f;
        for (int t = lane; t < T; t += 32) { float e = expf(r[t] - mx); r[t] = e; sum += e; }
        sum = espb::warp_sum(sum);
        for (int t = lane; t < T; t += 32) r[t] = r[t] / sum;
      }
      __syncthreads();
    }
    const float* tile = ring + (i % S) * TILE_F;
    {
      // ---- context: A = P (16 slot rows, clamped to W-1), B = V tile, K-dim = t (warp w takes the 8-frame k-step w of the tile)
      const int tb = (i - nt) * TR, rows = min(TR, T - tb);
      if (warp * 8 < rows) {
        const int t0 = tb + warp * 8 + t4, t1 = t0 + 4;
        uint32_t ah[4], al[4];
        split_tf32(t0 < T ? sc[sa * Tmax + t0] : 0.f, ah[0], al[0]);
        split_tf32(t0 < T ? sc[sb * Tmax + t0] : 0.f, ah[1], al[1]);
        split_tf32(t1 < T ? sc[sa * Tmax + t1] : 0.f, ah[2], al[2]);
        split_tf32(t1 < T ? sc[sb * Tmax + t1] : 0.f, ah[3], al[3]);
#pragma unroll
        for (int n8 = 0; n8 < 8; ++n8) {
          uint32_t bh[2], bl[2];
          split_tf32(tile[(warp * 8 + t4) * VST + n8 * 8 + g], bh[0], bl[0]);
          split_tf32(tile[(warp * 8 + t4 + 4) * VST + n8 * 8 + g], bh[1], bl[1]);
          mma3_tf32(acc[n8], ah, al, bh, bl);
        }
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  // ---- cross-warp reduction: red[warp][slot 16][d 64] (32 KB) in the ring, then split store of the W valid slots
  float* red = ring;
  static_assert(S * TILE_F >= 8 * 16 * DK, "reduction scratch must fit in the ring");
#pragma unroll
  for (int n8 = 0; n8 < 8; ++n8) {
    float* r0p = red + ((long long)warp * 16 + g) * DK + n8 * 8 + 2 * t4;
    float* r1p = red + ((long long)warp * 16 + g + 8) * DK + n8 * 8 + 2 * t4;
    r0p[0] = acc[n8][0]; r0p[1] = acc[n8][1];
    r1p[0] = acc[n8][2]; r1p[1] = acc[n8][3];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < W * DK; i += blockDim.x) {
    const int w = i / DK, d = i % DK;
    float a = 0.f;
#pragma unroll
    for (int ww = 0; ww < 8; ++ww) a += red[((long long)ww * 16 + w) * DK + d];
    store_split(ctx + ((long long)(u * Wall + w0 + w)) * D + h * DK + d, ctx_plane, a);
  }
}

#ifndef ESPB_SRC_ATTN_NW_DEFAULT
#define ESPB_SRC_ATTN_NW_DEFAULT 4
#endif
// ---------------------------------------------------------------- cross-attention, single pass (d_k = 64, beam <= 16, any T)
// Flash-decoding inside a block: K and V tiles of 64 frames stream TOGETHER through an S-deep cp.async ring (no [W][T] score buffer, so twice
// the bytes are in flight per SM and T is unbounded); warp w owns frames 8w..8w+7 of every tile and keeps its own online-softmax state
// (running max / partial sum per slot, partial context [16][64] in mma accumulators); the eight partial results are merged once at the end.
//   scores  C[16 slots][8 frames] = Q (A, split once into registers / smem) x K^T (B): every K element is read and split once
//   context O[16 slots][64]      += P (A = the C fragment re-used in place: the k index of the second product is simply a permutation of
//                                   the warp's 8 frames, lane t4 holds frames 2 t4, 2 t4 + 1) x V (B rows picked with the same permutation)
template <int S, int NW>   // NW warps per block, 8 NW frames per tile: NW = 4 -> four 57 KB blocks per SM, all U x H blocks of a 64 x 8 launch resident at once
__global__ void __launch_bounds__(NW * 32, 16 / NW) dec_src_attn_flash_kernel(const float* __restrict__ q, const float* __restrict__ kmem, const float* __restrict__ vmem,
                                                                    int Tmax, const int* __restrict__ lens, int W, int D, int H,
                                                                    float* __restrict__ ctx, long long ctx_plane, int w0, int Wall) {
  constexpr int DK = 64, QST = 68, ST = 68, TR = 8 * NW, TILE_F = TR * ST, STAGE_F = 2 * TILE_F;
  extern __shared__ float sm[];  // q lo [16][68] | ring [S][K [64][68] | V [64][68]] (reused for the cross-warp merge)
  espb::pdl_trigger();
  espb::pdl_wait();
  const int u = blockIdx.x / H, h = blockIdx.x % H;
  const int T = lens[u];
  float* qlo = sm;
  float* ring = qlo + 16 * QST;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const float4* kb = reinterpret_cast<const float4*>(kmem + ((long long)(u * H + h) * Tmax) * DK);
  const float4* vb = reinterpret_cast<const float4*>(vmem + ((long long)(u * H + h) * Tmax) * DK);
  const int nt = (T + TR - 1) / TR;
  auto issue = [&](int i) {
    if (i < nt) {
      const int tb = i * TR;
      float* dst = ring + (i % S) * STAGE_F;
#pragma unroll
      for (int j = threadIdx.x; j < 2 * TR * 16; j += NW * 32) {
        const int isv = j / (TR * 16), rr = (j >> 4) % TR, cc = j & 15;
        const bool ok = tb + rr < T;      // frames past the utterance are zero-filled (src-size 0)
        cp_async16_zfill(dst + isv * TILE_F + rr * ST + cc * 4, (isv ? vb : kb) + (ok ? (long long)(tb + rr) * 16 + cc : 0), ok ? 16 : 0);
      }
    }
    cp_async_commit();                    // one (possibly empty) group per tile index keeps the wait_group arithmetic uniform
  };
#pragma unroll
  for (int i = 0; i < S - 1; ++i) issue(i);
  // Q A-fragments: hi parts in registers, lo parts in shared memory (register budget: 128 per thread at two blocks per SM)
  uint32_t qh[8][4];
  {
    const float* qg = q + ((long long)(u * Wall + w0)) * D + h * DK;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = g + (e & 1) * 8, col = ks * 8 + t4 + (e >> 1) * 4;
        const float x = (row < W) ? __ldg(qg + (long long)row * D + col) : 0.f;
        uint32_t lo;
        split_tf32(x, qh[ks][e], lo);
        if (warp == 0) qlo[row * QST + col] = __uint_as_float(lo);
      }
    }
  }
  const float inv_rs = 0.125f;   // 1 / sqrt(d_k), exact
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float acc[8][4];
#pragma unroll
  for (int n8 = 0; n8 < 8; ++n8) { acc[n8][0] = 0.f; acc[n8][1] = 0.f; acc[n8][2] = 0.f; acc[n8][3] = 0.f; }
  const int f0 = warp * 8;

  for (int i = 0; i < nt; ++i) {
    cp_async_wait<S - 2>();               // this thread's copies of tile i have landed ...
    __syncthreads();                      // ... and everyone's (also orders the qlo writes before the first use); tile i-1's slot is refilled next
    issue(i + S - 1);
    const int tb = i * TR;
    if (tb + f0 >= T) continue;           // warp-uniform: none of this warp's frames exists
    const float* kt = ring + (i % S) * STAGE_F;
    const float* vt = kt + TILE_F;
    float c[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f}, c2[4] = {0.f, 0.f, 0.f, 0.f};
    const float* kr = kt + (f0 + g) * ST + t4;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      uint32_t bh[2], bl[2], al[4];
      split_tf32(kr[ks * 8], bh[0], bl[0]);
      split_tf32(kr[ks * 8 + 4], bh[1], bl[1]);
      al[0] = __float_as_uint(qlo[g * QST + ks * 8 + t4]); al[1] = __float_as_uint(qlo[(g + 8) * QST + ks * 8 + t4]);
      al[2] = __float_as_uint(qlo[g * QST + ks * 8 + t4 + 4]); al[3] = __float_as_uint(qlo[(g + 8) * QST + ks * 8 + t4 + 4]);
      mma_m16n8k8_tf32(c1, al, bh);
      mma_m16n8k8_tf32(c2, qh[ks], bl);
      mma_m16n8k8_tf32(c, qh[ks], bh);
    }
    // scores of slots g (c[0], c[1]) and g+8 (c[2], c[3]) for frames fa, fa+1; no memory mask beyond the utterance's own frames
    const int fa = tb + f0 + 2 * t4;
#pragma unroll
    for (int e = 0; e < 4; ++e) c[e] = (c[e] + (c1[e] + c2[e])) * inv_rs;
    if (fa >= T) { c[0] = -INFINITY; c[2] = -INFINITY; }
    if (fa + 1 >= T) { c[1] = -INFINITY; c[3] = -INFINITY; }
    float x0 = fmaxf(c[0], c[1]), x1 = fmaxf(c[2], c[3]);
    x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1));
    x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
    const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);          // finite: frame tb + f0 exists
    const float a0 = expf(m0 - n0), a1 = expf(m1 - n1);          // first tile: exp(-inf) = 0
    const float p0 = expf(c[0] - n0), p1 = expf(c[1] - n0), p2 = expf(c[2] - n1), p3 = expf(c[3] - n1);
    l0 = fmaf(l0, a0, p0 + p1); l1 = fmaf(l1, a1, p2 + p3);      // this lane's share of the row sums
    m0 = n0; m1 = n1;
    uint32_t ah[4], alo[4];
    split_tf32(p0, ah[0], alo[0]); split_tf32(p2, ah[1], alo[1]);   // A fragment: (row g, k t4) = frame 2 t4; (row g+8, k t4)
    split_tf32(p1, ah[2], alo[2]); split_tf32(p3, ah[3], alo[3]);   //             (row g, k t4+4) = frame 2 t4 + 1; (row g+8, k t4+4)
    const float* vr = vt + (f0 + 2 * t4) * ST + g;
#pragma unroll
    for (int n8 = 0; n8 < 8; ++n8) {
      acc[n8][0] *= a0; acc[n8][1] *= a0; acc[n8][2] *= a1; acc[n8][3] *= a1;
      uint32_t bh[2], bl[2];
      split_tf32(vr[n8 * 8], bh[0], bl[0]);            // B fragment: (k t4, n g) = V[frame 2 t4][8 n8 + g]
      split_tf32(vr[ST + n8 * 8], bh[1], bl[1]);       //             (k t4+4, n g) = V[frame 2 t4 + 1][8 n8 + g]
      mma3_tf32(acc[n8], ah, alo, bh, bl);
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  // ---- merge of the NW warps: red[warp][slot 16][66] = (O[64], m, l) in the ring
  float* red = ring;
  static_assert(S * STAGE_F >= NW * 16 * 66, "merge scratch must fit in the ring");
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
#pragma unroll
  for (int n8 = 0; n8 < 8; ++n8) {
    float* r0p = red + ((long long)warp * 16 + g) * 66 + n8 * 8 + 2 * t4;
    float* r1p = red + ((long long)warp * 16 + g + 8) * 66 + n8 * 8 + 2 * t4;
    r0p[0] = acc[n8][0]; r0p[1] = acc[n8][1];
    r1p[0] = acc[n8][2]; r1p[1] = acc[n8][3];
  }
  if (t4 == 0) {
    red[((long long)warp * 16 + g) * 66 + 64] = m0; red[((long long)warp * 16 + g) * 66 + 65] = l0;
    red[((long long)warp * 16 + g + 8) * 66 + 64] = m1; red[((long long)warp * 16 + g + 8) * 66 + 65] = l1;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < W * DK; i += blockDim.x) {
    const int w = i / DK, d = i % DK;
    float M = -INFINITY;
#pragma unroll
    for (int ww = 0; ww < NW; ++ww) M = fmaxf(M, red[((long long)ww * 16 + w) * 66 + 64]);
    float L = 0.f, a = 0.f;
#pragma unroll
    for (int ww = 0; ww < NW; ++ww) {
      const float* r = red + ((long long)ww * 16 + w) * 66;
      const float e = expf(r[64] - M);      // a warp without frames: exp(-inf) = 0
      L = fmaf(r[65], e, L);
      a = fmaf(r[d], e, a);
    }
    store_split(ctx + ((long long)(u * Wall + w0 + w)) * D + h * DK + d, ctx_plane, a / L);
  }
}

// ---------------------------------------------------------------- row-wise top-k (descending; ties -> lower index)
// vals[r][k], ids[r][k] from x[r][0..V) * scale.  One block per row; every thread keeps its V/256 values in registers and the
// block runs k rounds of arg-max (winner knocked out by its owner).  V <= 256 * NV.
template <int NV>
__global__ void __launch_bounds__(256) rows_topk_kernel(const float* __restrict__ x, long long ld, int V, float scale, int k,
                                                        int* __restrict__ ids, float* __restrict__ vals) {
  __shared__ float bv[8]; __shared__ int bi[8];
  __shared__ int win_idx;
  const float* r = x + (long long)blockIdx.x * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = threadIdx.x + i * 256;
    v[i] = (c < V) ? r[c] * scale : -INFINITY;
  }
  for (int round = 0; round < k; ++round) {
    float best = -INFINITY; int idx = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = threadIdx.x + i * 256;
      if (v[i] > best) { best = v[i]; idx = c; }   // ascending c within a thread: first maximum wins
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
      if (ov > best || (ov == best && oi < idx)) { best = ov; idx = oi; }
    }
    if (lane == 0) { bv[warp] = best; bi[warp] = idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float bb = bv[0]; int id = bi[0];
      for (int w = 1; w < 8; ++w)
        if (bv[w] > bb || (bv[w] == bb && bi[w] < id)) { bb = bv[w]; id = bi[w]; }
      win_idx = id;
      ids[(long long)blockIdx.x * k + round] = id;
      vals[(long long)blockIdx.x * k + round] = bb;
    }
    __syncthreads();
    const int wi = win_idx;
#pragma unroll
    for (int i = 0; i < NV; ++i) if (threadIdx.x + i * 256 == wi) v[i] = -INFINITY;
  }
}

// ---------------------------------------------------------------- CTC prefix scorer
// Initial state (ctc_prefix_score.py:86-95): r[t][0] = logzero, r[t][1] = cumsum_t x[t][blank]; s_prev = 0.
__global__ void ctc_init_state_kernel(const float* __restrict__ logp, int Tmax, int V, const int* __restrict__ lens, int blank, int W, int n,
                                      float* __restrict__ r, float* __restrict__ s_prev) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int u = s / W;
  const int T = lens[u];
  float4* rr = reinterpret_cast<float4*>(r) + (long long)s * Tmax;
  float c = 0.f;
  for (int t = 0; t < Tmax; ++t) {
    if (t < T) c += logp[((long long)u * Tmax + t) * V + blank];
    const float rb = (t < T) ? c : LOGZERO;
    rr[t] = make_float4(LOGZERO, rb, logaddexp(LOGZERO, rb), 0.f);
  }
  s_prev[s] = 0.f;
}

// Streaming extension of a prefix state to a longer encoder output (CTCPrefixScoreTH.extend_state, ctc_prefix_score.py:251-270; Eq. 14 of
// arXiv:2006.14941): frames [0, T_old) are kept; for the new frames the prefix can only be continued by blanks:
// r^n[t] = logzero, r^b[t] = r^b[t-1] + x[t][blank].  One thread per state, sequential over the (few) new frames like the reference's loop.
__global__ void ctc_extend_state_kernel(const float* __restrict__ logp, int T_new, int V, int blank, int n, const float* __restrict__ r_old, int T_old,
                                        float* __restrict__ r_new) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const float4* ro = reinterpret_cast<const float4*>(r_old) + (long long)s * T_old;
  float4* rn = reinterpret_cast<float4*>(r_new) + (long long)s * T_new;
  const int keep = min(T_old, T_new);
  for (int t = 0; t < keep; ++t) rn[t] = ro[t];
  float rb = keep > 0 ? ro[keep - 1].y : LOGZERO;
  for (int t = max(keep, 1); t < T_new; ++t) {
    rb += logp[(long long)t * V + blank];
    rn[t] = make_float4(LOGZERO, rb, logaddexp(LOGZERO, rb), 0.f);
  }
  if (keep == 0 && T_new > 0) rn[0] = make_float4(LOGZERO, LOGZERO, logaddexp(LOGZERO, LOGZERO), 0.f);
}

// log_phi[t] of the previous state: r_sum unless the candidate repeats the last label (ctc_prefix_score.py:135-144).
// State layout: float4 per frame (r^n, r^b, r_sum = logaddexp(r^n, r^b), 0) so that scoring needs no transcendental for log_phi.
__device__ __forceinline__ float ctc_phi(const float4* __restrict__ rp, int t, bool same) {
  const float4 v = __ldg(rp + t);
  return same ? v.y : v.z;
}

// log_psi of extending the prefix of a slot by token c (ctc_prefix_score.py:166-189).  It depends only on the PREVIOUS state:
//   log_psi = logsumexp( {log_phi[t-1] + x[t,c]}_{t=start..T-1}, r[start-1,0] ),   r[start-1,0] = x[0,c] if the prefix is empty else logzero
// so it is a reduction over t: one warp per (slot, candidate), lanes stride t.  Must be called by a full warp.
__device__ __forceinline__ float ctc_log_psi_warp(const float* __restrict__ x, long long st_t, long long st_c, int T, int blank, int eos,
                                                  const float4* __restrict__ rp, int c, int last, int out_len, int lane) {
  if (T <= 0) return LOGZERO;                                              // empty encoder output (refused on the host; never index rp[-1])
  if (c == eos) return __ldg(rp + (T - 1)).z;                             // (:184-185) r_sum[T-1]
  if (c == blank) return LOGZERO;                                          // (:187-189)
  const int start = max(out_len, 1);
  const bool same = (c == last);
  float m = -INFINITY, ssum = 0.f;   // per-lane streaming log-sum-exp, merged across the warp at the end
  const float* xc = x + c * st_c;
  auto term = [&](int t) { return ctc_phi(rp, t - 1, same) + __ldg(xc + t * st_t); };
  auto fold = [&](float e) { if (e > m) { ssum = ssum * expf(m - e) + 1.f; m = e; } else { ssum += expf(e - m); } };
  int t = start + lane;
  for (; t + 96 < T; t += 128) {     // four frames per lane at a time: the eight loads are issued together, the folds keep their order
    const float e0 = term(t), e1 = term(t + 32), e2 = term(t + 64), e3 = term(t + 96);
    fold(e0); fold(e1); fold(e2); fold(e3);
  }
  for (; t < T; t += 32) fold(term(t));
  if (lane == 0) {   // the r[start-1,0] term
    const float r0 = (out_len == 0) ? x[c * st_c] : LOGZERO;
    if (r0 > m) { ssum = ssum * expf(m - r0) + 1.f; m = r0; } else { ssum += expf(r0 - m); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, ssum, o);
    const float nm = fmaxf(m, om);
    ssum = (m == -INFINITY ? 0.f : ssum * expf(m - nm)) + (om == -INFINITY ? 0.f : os * expf(om - nm));
    m = nm;
  }
  return m + logf(ssum);
}

// Scores for candidate lists: cand [n][P] (from the pre-beam) plus eos as candidate P. Outputs part[n][P+1] = log_psi - s_prev
// and psi[n][P+1]. Duplicate eos (eos already among the P) is flagged by valid[n][P+1] = 0.  One warp per (slot, candidate).
__global__ void __launch_bounds__(256) ctc_score_cands_kernel(const float* __restrict__ logp, int Tmax, int V, const int* __restrict__ lens, int blank,
                                                              int eos, int W, int n, const float* __restrict__ r_prev, const float* __restrict__ s_prev,
                                                              const int* __restrict__ last_tok, int out_len, const int* __restrict__ step_ptr,
                                                              const int* __restrict__ cand, int P, float* __restrict__ part,
                                                              float* __restrict__ psi, int* __restrict__ valid, int token_major) {
  if (step_ptr) out_len += *step_ptr;
  const int idx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (idx >= n * (P + 1)) return;
  const int s = idx / (P + 1), j = idx % (P + 1);
  const int u = s / W;
  const int c = (j < P) ? cand[(long long)s * P + j] : eos;
  int ok = 1;
  if (j == P) for (int q = 0; q < P; ++q) if (cand[(long long)s * P + q] == eos) ok = 0;
  // token_major: logp is [u][v][t] (a candidate's column is contiguous in t -> coalesced); else [u][t][v]
  const float v = ctc_log_psi_warp(logp + (long long)u * Tmax * V, token_major ? 1 : V, token_major ? Tmax : 1, lens[u], blank, eos,
                                   reinterpret_cast<const float4*>(r_prev) + (long long)s * Tmax, c, last_tok[s], out_len, lane);
  if (lane == 0) { psi[idx] = v; part[idx] = v - s_prev[s]; valid[idx] = ok; }
}

// Dense variant (ctc_weight == 1: no pre-beam, ctc_prefix_score.py:118-122): part[n][V].  One thread per (slot, token); adjacent
// threads read adjacent tokens of a frame (coalesced), streaming log-sum-exp over t.
__global__ void __launch_bounds__(128) ctc_score_dense_kernel(const float* __restrict__ logp, int Tmax, int V, const int* __restrict__ lens, int blank,
                                                              int eos, int W, int n, const float* __restrict__ r_prev, const float* __restrict__ s_prev,
                                                              const int* __restrict__ last_tok, int out_len, float* __restrict__ part) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n * V) return;
  const int s = (int)(idx / V), c = (int)(idx % V);
  const int u = s / W, T = lens[u];
  const float* x = logp + (long long)u * Tmax * V;
  const float4* rp = reinterpret_cast<const float4*>(r_prev) + (long long)s * Tmax;
  float v;
  if (T <= 0) v = LOGZERO;
  else if (c == eos) v = __ldg(rp + (T - 1)).z;
  else if (c == blank) v = LOGZERO;
  else {
    const int start = max(out_len, 1);
    const bool same = (c == last_tok[s]);
    float m = (out_len == 0) ? x[c] : LOGZERO, ssum = 1.f;
    for (int t = start; t < T; ++t) {
      const float e = ctc_phi(rp, t - 1, same) + x[(long long)t * V + c];
      if (e > m) { ssum = ssum * expf(m - e) + 1.f; m = e; } else { ssum += expf(e - m); }
    }
    v = m + logf(ssum);
  }
  part[idx] = v - s_prev[s];
}

// ---------------------------------------------------------------- beam selection + post-process, one warp per utterance
struct BeamState {
  // per slot (n = U*W), "cur" read / "nxt" written
  const float* score; const float* sc_dec; const float* sc_ctc; const int* active;
  float* n_score; float* n_sc_dec; float* n_sc_ctc; int* n_active; int* n_last_tok;
  int* n_parent;      // [n] parent slot of each new slot (ancestor-table / CTC-state gathers)
  int* bp_parent; int* bp_token;   // [maxlen][n] back-pointers for sequence reconstruction
  // ended hypotheses: per utterance append (step, slot, score, dec, ctc)
  int* ended_count; int* ended_step; int* ended_slot; float* ended_score; float* ended_dec; float* ended_ctc; int ended_cap;
  float* best_at_step;  // [U][maxlen_cap] best ended score per step (end detection)
  float* best_all;      // [U]
  int* utt_done;        // [U]
};

// mode 0: decoder only      -- cand_val[n][P] = w_dec*logp of cand_ids; total = (val + penalty) + score
// mode 1: joint             -- candidates j<P from the pre-beam + eos as candidate P; part/valid [n][P+1]
//                              total = ((dec + penalty) + w_ctc*part) + score   (batch_beam_search.py:293-309)
// mode 2: CTC only (dense)  -- cand_val[n][P] = w_ctc*part of cand_ids, part = dense [n][V]
template <int MAXC, int NT>   // each thread owns candidates tid, tid+NT, ...: supports W*PC <= NT*MAXC; NT = 32 (one warp) or 256 (wide beams)
__global__ void __launch_bounds__(NT) beam_select_kernel(BeamState st, int U, int W, int P, int V, int step, const int* __restrict__ step_ptr,
                                                         const int* __restrict__ maxlen,
                                                         const int* __restrict__ minlen, int eos, float w_dec, float w_ctc, float penalty, int mode,
                                                         const int* __restrict__ cand_ids, const float* __restrict__ cand_val,
                                                         const float* __restrict__ logp_dec /* [n][V] or null */, const float* __restrict__ part,
                                                         const int* __restrict__ valid, int end_detect, int maxlen_cap) {
  if (step_ptr) step += *step_ptr;
  const int u = blockIdx.x, lane = threadIdx.x;   // `lane`: thread index within the block (a warp for NT = 32)
  __shared__ float red_v[NT / 32];
  __shared__ int red_i[NT / 32];
  const int PC = (mode == 1) ? P + 1 : P;   // candidates per slot
  const int total = W * PC;
  float tot[MAXC];
  const bool done = st.utt_done[u] != 0;
#pragma unroll
  for (int q = 0; q < MAXC; ++q) {
    const int ci = lane + q * NT;
    float t = -INFINITY;
    if (ci < total && !done) {
      const int w = ci / PC, j = ci % PC, s = u * W + w;
      if (st.active[s]) {
        if (mode == 1) {
          if (valid[(long long)s * PC + j]) {
            const float dec = (j < P) ? cand_val[(long long)s * P + j] : w_dec * logp_dec[(long long)s * V + eos];
            t = ((dec + penalty) + w_ctc * part[(long long)s * PC + j]) + st.score[s];
          }
        } else {
          t = (cand_val[(long long)s * P + j] + penalty) + st.score[s];
        }
      }
    }
    tot[q] = t;
  }
  const int mlen = maxlen[u];
  const bool last_step = (step == mlen - 1);
  float step_best = -INFINITY;
  for (int k = 0; k < W; ++k) {
    // warp arg-max over the remaining candidates (ties -> lower flat index)
    float best = -INFINITY; int bidx = 0x7fffffff;
#pragma unroll
    for (int q = 0; q < MAXC; ++q) {
      const int ci = lane + q * NT;
      if (tot[q] > best) { best = tot[q]; bidx = ci; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (ov > best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
    }
    if (NT > 32) {   // across the warps of the block: every thread ends up with the same winner
      __syncthreads();
      if ((lane & 31) == 0) { red_v[lane >> 5] = best; red_i[lane >> 5] = bidx; }
      __syncthreads();
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) {
        const float ov = red_v[w];
        const int oi = red_i[w];
        if (ov > best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
      }
    }
    const int ns = u * W + k;
    const long long bp = (long long)step * U * W + ns;
    if (best == -INFINITY) {                // fewer candidates than beam slots (utterance finished)
      if (lane == 0) {
        st.n_active[ns] = 0; st.n_score[ns] = 0.f; st.n_sc_dec[ns] = 0.f; st.n_sc_ctc[ns] = 0.f; st.n_last_tok[ns] = eos;
        st.n_parent[ns] = ns; st.bp_parent[bp] = -1; st.bp_token[bp] = eos;
      }
      continue;
    }
#pragma unroll
    for (int q = 0; q < MAXC; ++q) if (lane + q * NT == bidx) tot[q] = -INFINITY;   // remove the winner
    if (lane == 0) {
      const int w = bidx / PC, j = bidx % PC, s = u * W + w;
      const int tok = (mode == 1 && j == P) ? eos : cand_ids[(long long)s * P + j];
      float dlogp = 0.f, cpart = 0.f;
      if (mode != 2) dlogp = logp_dec[(long long)s * V + tok];
      if (mode == 1) cpart = part[(long long)s * PC + j];
      if (mode == 2) cpart = part[(long long)s * V + tok];
      const float ndec = st.sc_dec[s] + dlogp, nctc = st.sc_ctc[s] + cpart;
      st.bp_parent[bp] = s; st.bp_token[bp] = tok;
      st.n_parent[ns] = s;
      st.n_score[ns] = best; st.n_sc_dec[ns] = ndec; st.n_sc_ctc[ns] = nctc; st.n_last_tok[ns] = tok;
      const bool ended = last_step || tok == eos;   // last step: eos is appended to every hypothesis (batch_beam_search.py:392-407)
      st.n_active[ns] = ended ? 0 : 1;
      if (ended && step >= minlen[u]) {
        const int e = st.ended_count[u];
        if (e < st.ended_cap) {
          const long long o = (long long)u * st.ended_cap + e;
          st.ended_step[o] = step; st.ended_slot[o] = ns; st.ended_score[o] = best; st.ended_dec[o] = ndec; st.ended_ctc[o] = nctc;
          st.ended_count[u] = e + 1;
        }
        step_best = fmaxf(step_best, best);
      }
    }
  }
  if (lane == 0 && !done) {
    if (end_detect) {
      // end_detect(ended, i) (e2e_asr_common.py:14-44): hypotheses with len(yseq) == i-m ended at step i-m-2
      if (step < maxlen_cap) st.best_at_step[(long long)u * maxlen_cap + step] = step_best;
      const float ball = fmaxf(st.best_all[u], step_best);
      st.best_all[u] = ball;
      int count = 0;
      for (int m = 0; m < 3; ++m) {
        const int j = step - m - 2;
        if (j >= 0 && j < maxlen_cap) {
          const float bs = st.best_at_step[(long long)u * maxlen_cap + j];
          if (bs > -INFINITY && bs - ball < -10.0f) ++count;
        }
      }
      if (count == 3) st.utt_done[u] = 1;
    }
    if (last_step) st.utt_done[u] = 1;
  }
}

// After selection: rows of the ancestor table and CTC states follow their parents.
__global__ void anc_update_kernel(const int* __restrict__ anc, int* __restrict__ n_anc, int anc_ld, const int* __restrict__ parent, int pos,
                                  const int* __restrict__ step_ptr, int n) {
  if (step_ptr) pos += *step_ptr;
  const int s = blockIdx.x;
  const int p = parent[s];
  for (int j = threadIdx.x; j < pos; j += blockDim.x) n_anc[(long long)s * anc_ld + j] = anc[(long long)p * anc_ld + j];
  if (threadIdx.x == 0) n_anc[(long long)s * anc_ld + pos] = p;
}

__device__ __forceinline__ float logaddexp_fast(float a, float b) {
  const float m = fmaxf(a, b);
  return m + __logf(__expf(a - m) + __expf(b - m));
}

// New CTC forward variables of each surviving slot: the recursion of ctc_prefix_score.py:128-164 for (parent state, chosen token),
// storing r[t][0..1].  One warp per slot: lanes prefetch 32 frames of (log_phi, x[t,c], x[t,blank]) in parallel, then the warp walks
// the 32 sequential steps with shuffles (the dependent chain is two logaddexp per frame); lane l keeps frame l for a coalesced store.
__global__ void __launch_bounds__(128) ctc_advance_kernel(const float* __restrict__ logp, int Tmax, int V, const int* __restrict__ lens, int blank, int eos,
                                                          int W, int n, const float* __restrict__ r_prev, const int* __restrict__ parent,
                                                          const int* __restrict__ par_last_tok, const int* __restrict__ new_tok,
                                                          const int* __restrict__ new_active, int out_len, const int* __restrict__ step_ptr,
                                                          float* __restrict__ r_new, float* __restrict__ s_new, int token_major) {
  if (step_ptr) out_len += *step_ptr;
  const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (s >= n) return;
  const int u = s / W;
  float4* ro = reinterpret_cast<float4*>(r_new) + (long long)s * Tmax;
  const float4 Z4 = make_float4(LOGZERO, LOGZERO, logaddexp(LOGZERO, LOGZERO), 0.f);
  const int c = new_tok[s];
  if (!new_active[s] || c == eos || c == blank) {   // ended / inactive hypotheses never use their state again
    for (int t = lane; t < Tmax; t += 32) ro[t] = Z4;
    if (lane == 0) s_new[s] = (new_active[s] && c == blank) ? LOGZERO : 0.f;   // log_psi[blank] = logzero (ctc_prefix_score.py:187-189)
    return;
  }
  const int p = parent[s], T = lens[u];
  const float* x = logp + (long long)u * Tmax * V;
  const long long st_t = token_major ? 1 : V, st_c = token_major ? Tmax : 1;
  const float4* rp = reinterpret_cast<const float4*>(r_prev) + (long long)p * Tmax;
  const int last = par_last_tok[p];
  const bool same = (c == last);
  const int start = max(out_len, 1);
  float rn = (out_len == 0) ? x[c * st_c] : LOGZERO, rb = LOGZERO;   // r[start-1]
  // a prefix longer than the encoder output (start - 1 >= T) has no valid frame left: the state is all-logzero (the reference's
  // r[start - 1] raises an IndexError there, ctc_prefix_score.py:147; the host reports it per utterance after the search)
  for (int t = lane; t < min(start - 1, Tmax); t += 32) ro[t] = Z4;
  if (lane == 0 && start - 1 < Tmax) ro[start - 1] = (start - 1 < T) ? make_float4(rn, rb, logaddexp(rn, rb), 0.f) : Z4;
  for (int t0 = start; t0 < T; t0 += 32) {
    const int t = t0 + lane;
    float phi = LOGZERO, xc = 0.f, xb = 0.f;
    if (t < T) { phi = ctc_phi(rp, t - 1, same); xc = x[t * st_t + c * st_c]; xb = x[t * st_t + blank * st_c]; }
    float my_n = LOGZERO, my_b = LOGZERO;
    const int cnt = min(32, T - t0);
    for (int i = 0; i < cnt; ++i) {
      const float ph = __shfl_sync(0xffffffffu, phi, i), c1 = __shfl_sync(0xffffffffu, xc, i), b1 = __shfl_sync(0xffffffffu, xb, i);
      // The two log-add-exp of a frame are the whole critical path of this kernel (T sequential frames): ex2 / lg2 approximations
      // (2 ulp) instead of expf / logf cut the dependent chain from ~25 to ~8 instructions; the error stays ~1e-7 relative per frame.
      const float nrn = logaddexp_fast(rn, ph) + c1;
      const float nrb = logaddexp_fast(rn, rb) + b1;
      rn = nrn; rb = nrb;
      if (lane == i) { my_n = rn; my_b = rb; }
    }
    if (t < T) ro[t] = make_float4(my_n, my_b, logaddexp(my_n, my_b), 0.f);
  }
  for (int t = T + lane; t < Tmax; t += 32) ro[t] = Z4;
  const float psi = ctc_log_psi_warp(x, st_t, st_c, T, blank, eos, rp, c, last, out_len, lane);
  if (lane == 0) s_new[s] = psi;
}

// CTC posteriors [u][t][v] -> [u][v][t]: the per-step candidate scoring / state advance read whole token columns.
__global__ void __launch_bounds__(256) transpose_tv_kernel(const float* __restrict__ x, int Tmax, int V, float* __restrict__ xt) {
  __shared__ float tile[32][33];
  const long long base = (long long)blockIdx.z * Tmax * V;
  const int v0 = blockIdx.x * 32, t0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, v = v0 + threadIdx.x;
    tile[i][threadIdx.x] = (t < Tmax && v < V) ? x[base + (long long)t * V + v] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int v = v0 + i, t = t0 + threadIdx.x;
    if (v < V && t < Tmax) xt[base + (long long)v * Tmax + t] = tile[threadIdx.x][i];
  }
}

__global__ void step_inc_kernel(int* step) { *step += 1; }

// ---------------------------------------------------------------- LM shallow fusion helpers (espnet2/lm/transformer_lm.py, beam_search.py:264-293)
// Embedding rows of the newest tokens as a split [2][n][E] GEMM operand (TransformerLM.embed, then encoder.embed[0] = Linear).
__global__ void gather_rows_split_kernel(const int* __restrict__ tok, const float* __restrict__ emb, int E, float* __restrict__ out, long long plane) {
  espb::pdl_trigger();
  espb::pdl_wait();
  const int s = blockIdx.x;
  const float* e = emb + (long long)tok[s] * E;
  for (int c = threadIdx.x; c < E; c += blockDim.x) store_split(out + (long long)s * E + c, plane, e[c]);
}
// encoder.embed[3..4]: ReLU, then PositionalEncoding x * sqrt(D) + pe[pos] (embedding.py:85-95) or identity (pos_enc None), in place.
__global__ void relu_posenc_kernel(float* __restrict__ x, int D, const float* __restrict__ pe, int pos, const int* __restrict__ step_ptr, float scale) {
  espb::pdl_trigger();
  espb::pdl_wait();
  if (step_ptr) pos += *step_ptr;
  const int s = blockIdx.x;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float v = fmaxf(x[(long long)s * D + c], 0.f);
    if (pe) v = v * scale + pe[(long long)pos * D + c];
    x[(long long)s * D + c] = v;
  }
}
// weighted sum of two score matrices as the reference forms it: (wa * a) + (wb * b), each product rounded (no fma)
__global__ void axpby_kernel(const float* __restrict__ a, float wa, const float* __restrict__ b, float wb, float* __restrict__ out, long long n) {
  espb::pdl_trigger();
  espb::pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __fadd_rn(__fmul_rn(wa, a[i]), __fmul_rn(wb, b[i]));
}
// per-scorer running scores of the new hypotheses (merge_scores, beam_search.py:264-293): new[ns] = prev[parent[ns]] + logp[parent[ns]][tok[ns]],
// also recorded per step so that ended hypotheses can be read back.  a / b: two full scorers (decoder, lm); b may be null.
__global__ void track_scores_kernel(const int* __restrict__ parent, const int* __restrict__ tok, const int* __restrict__ bp_parent,
                                    const float* __restrict__ logp_a, const float* __restrict__ logp_b, int V, const float* __restrict__ prev_a,
                                    const float* __restrict__ prev_b, float* __restrict__ new_a, float* __restrict__ new_b, float* __restrict__ hist_a,
                                    float* __restrict__ hist_b, int step, const int* __restrict__ step_ptr, int n) {
  if (step_ptr) step += *step_ptr;
  const int ns = blockIdx.x * blockDim.x + threadIdx.x;
  if (ns >= n) return;
  float va = 0.f, vb = 0.f;
  if (bp_parent[(long long)step * n + ns] >= 0) {
    const int p = parent[ns], t = tok[ns];
    if (logp_a) va = prev_a[p] + logp_a[(long long)p * V + t];
    if (logp_b) vb = prev_b[p] + logp_b[(long long)p * V + t];
  }
  if (logp_a) { new_a[ns] = va; hist_a[(long long)step * n + ns] = va; }
  if (logp_b) { new_b[ns] = vb; hist_b[(long long)step * n + ns] = vb; }
}

// ---------------------------------------------------------------- LSTM LM (espnet2/lm/seq_rnn_lm.py: Embedding -> nn.LSTM -> Linear)
// Recurrent state ring h, c [2][L][n][Hp]: step pos reads its parent from ring (pos-1)&1 at slot anc[s][pos-1] and writes ring pos&1 at
// slot s (zeros at pos 0).  Layer l's GEMM operand is the split [2][n][Kp_l] = [input | parent h]: Kp_0 = Ep + Hp, Kp_l = 2 Hp; the
// operands lie back to back in one buffer.  Pad columns are never written here (the host zeroes them once).
__device__ __forceinline__ int rnnlm_parent(const int* anc, int anc_ld, int pos, int s) {
  return pos > 0 ? anc[(long long)s * anc_ld + pos - 1] : -1;
}

// Embedding row of the newest token -> layer 0's input half; every layer's parent h -> that layer's recurrent half.
__global__ void rnnlm_gather_kernel(const int* __restrict__ tok, const float* __restrict__ emb, int E, int Ep, const int* __restrict__ anc,
                                    int anc_ld, int pos, const int* __restrict__ step_ptr, const float* __restrict__ h_ring, int L, int n, int H,
                                    int Hp, float* __restrict__ xs) {
  espb::pdl_trigger();
  espb::pdl_wait();
  if (step_ptr) pos += *step_ptr;
  const int s = blockIdx.x;
  const long long kp0 = Ep + Hp, kp1 = 2LL * Hp;
  const float* e = emb + (long long)tok[s] * E;
  for (int c = threadIdx.x; c < E; c += blockDim.x) store_split(xs + s * kp0 + c, n * kp0, e[c]);
  const int p = rnnlm_parent(anc, anc_ld, pos, s);
  const float* hp = h_ring + (long long)((pos - 1) & 1) * L * n * Hp;
  for (int l = 0; l < L; ++l) {
    const long long kp = l ? kp1 : kp0;
    float* x = xs + (l ? 2LL * n * kp0 + 2LL * (l - 1) * n * kp1 : 0LL) + s * kp + (l ? Hp : Ep);
    const float* src = hp + ((long long)l * n + (p < 0 ? 0 : p)) * Hp;
    for (int c = threadIdx.x; c < H; c += blockDim.x) store_split(x + c, n * kp, p < 0 ? 0.f : src[c]);
  }
}

__device__ __forceinline__ float sigmoid_acc(float v) { return 1.f / (1.f + expf(-v)); }

// gates [n][4H] (i, f, g, o, biases included) + parent c -> c' = σ(f) c + σ(i) tanh(g), h' = σ(o) tanh(c') into ring pos&1 (plain), and h'
// split into the next consumer's operand out[s * out_ld + j].
__global__ void lstm_cell_kernel(const float* __restrict__ gates, const int* __restrict__ anc, int anc_ld, int pos, const int* __restrict__ step_ptr,
                                 float* __restrict__ h_ring, float* __restrict__ c_ring, int layer, int L, int n, int H, int Hp,
                                 float* __restrict__ out, long long out_plane, int out_ld) {
  espb::pdl_trigger();
  espb::pdl_wait();
  if (step_ptr) pos += *step_ptr;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * H) return;
  const int s = (int)(i / H), j = (int)(i % H);
  const float* g = gates + (long long)s * 4 * H + j;
  const int p = rnnlm_parent(anc, anc_ld, pos, s);
  const float cp = p < 0 ? 0.f : c_ring[((long long)((pos - 1) & 1) * L + layer) * n * Hp + (long long)p * Hp + j];
  const float c = sigmoid_acc(g[H]) * cp + sigmoid_acc(g[0]) * tanhf(g[2 * H]);
  const float h = sigmoid_acc(g[3 * H]) * tanhf(c);
  const long long o = ((long long)(pos & 1) * L + layer) * n * Hp + (long long)s * Hp + j;
  h_ring[o] = h;
  c_ring[o] = c;
  store_split(out + (long long)s * out_ld + j, out_plane, h);
}

__global__ void count_active_kernel(const int* __restrict__ active, int n, int* __restrict__ out) {
  __shared__ float red[33];
  float c = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) c += active[i] ? 1.f : 0.f;
  c = espb::block_sum(c, red);
  if (threadIdx.x == 0) out[0] = (int)c;
}

}  // namespace

extern "C" {

int espb_dec_embed_f32(const int* last_tok, const float* emb, const float* pe, int pos, const int* step_ptr, int n, int D, float scale, float* x,
                       cudaStream_t stream) {
  espb::launch_pdl(dec_embed_kernel, dim3(n), dim3(128), 0, stream, last_tok, emb, pe, pos, step_ptr, D, scale, x);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_dec_self_attn_f32(const float* qkv, float* kc, float* vc, const int* anc, int anc_ld, int n, int D, int H, int pos, const int* step_ptr,
                           int max_pos, float* ctx, long long ctx_plane, cudaStream_t stream) {
  const int warps = 4;
  const int sc_ld = (step_ptr ? max_pos : pos) + 1;   // with a device-side step the score buffer is sized for the longest prefix
  const size_t smem = (size_t)warps * sc_ld * sizeof(float);
  if (smem > 48 * 1024) { espb_set_error("dec_self_attn: prefix too long for the score buffer"); return ESPB_ERR_ARG; }
  const bool fast64 = (D / H == 64) && (D % 4 == 0) && (ctx_plane % 4 == 0) && ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(kc) |
                       reinterpret_cast<uintptr_t>(vc) | reinterpret_cast<uintptr_t>(ctx)) & 15) == 0 && !getenv("ESPB_SELF_ATTN_GENERIC");
  if (fast64)
    espb::launch_pdl(dec_self_attn64_kernel, dim3((n * H + warps - 1) / warps), dim3(warps * 32), smem, stream, qkv, kc, vc, anc, anc_ld, n, D, H, pos,
                     step_ptr, sc_ld, ctx, ctx_plane);
  else
    espb::launch_pdl(dec_self_attn_kernel, dim3((n * H + warps - 1) / warps), dim3(warps * 32), smem, stream, qkv, kc, vc, anc, anc_ld, n, D, H, pos,
                     step_ptr, sc_ld, ctx, ctx_plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_dec_src_attn_f32(const float* q, const float* kmem, const float* vmem, int U, int Tmax, const int* lens, int W, int D, int H, float* ctx,
                          long long ctx_plane, cudaStream_t stream) {
  const int dk = D / H;
  if (W > 64 || dk > 128 || (dk & 3)) { espb_set_error("dec_src_attn: needs beam <= 64 and d_k a multiple of 4, <= 128"); return ESPB_ERR_ARG; }
  int lpr = 1;
  while (lpr * 4 < dk) lpr <<= 1;
  for (int w0 = 0; w0 < W; w0 += 16) {   // the kernels keep <= 16 beam slots per block; wider beams stream K/V once per group of 16
    const int Wg = (W - w0 < 16) ? W - w0 : 16;
    if (dk == 64 && !getenv("ESPNET_B200_SRC_ATTN_FFMA") && !getenv("ESPNET_B200_SRC_ATTN_TWOPASS")) {
      // single-pass kernel: 3 stages of (K, V) tiles = 112 KB -> two blocks per SM, 128 KB of loads in flight per SM
      using FlashFn = void (*)(const float*, const float*, const float*, int, const int*, int, int, int, float*, long long, int, int);
      // NW = 4 (default): four 57 KB blocks per SM -- 528 resident on an H100's 132 SMs, so a 64-utterance x 8-head launch is one wave; NW = 8
      // (ESPB_SRC_ATTN_NW=8, the first version): two 112 KB blocks per SM.  Same bytes in flight per SM.
      static int nw = 0;
      if (!nw) { const char* e = getenv("ESPB_SRC_ATTN_NW"); nw = (e && e[0] == '8') ? 8 : (e && e[0] == '4') ? 4 : ESPB_SRC_ATTN_NW_DEFAULT; }
      const FlashFn fn = (nw == 4) ? dec_src_attn_flash_kernel<3, 4> : dec_src_attn_flash_kernel<3, 8>;
      const size_t smem = (16 * 68 + 3 * 2 * 8 * nw * 68) * sizeof(float);
      static bool attr = false;
      if (!attr) {
        if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
          espb_set_error("dec_src_attn: cannot raise dynamic shared memory"); return ESPB_ERR_CUDA;
        }
        attr = true;
      }
      espb::launch_pdl(fn, dim3(U * H), dim3(nw * 32), smem, stream, q, kmem, vmem, Tmax, lens, Wg, D, H, ctx, ctx_plane, w0, W);
      ESPB_CHECK_LAUNCH();
      continue;
    }
    if (dk == 64 && !getenv("ESPNET_B200_SRC_ATTN_FFMA")) {   // two-pass variant (scores of the whole utterance in smem), kept for A/B
      const size_t scs4 = ((size_t)Wg * Tmax + 3) & ~(size_t)3;
      const size_t fixed = (16 * 68 + scs4) * sizeof(float), tile_b = 64 * 72 * sizeof(float);
      // deepest ring that still lets two blocks share an SM (227 KB), else the deepest that fits one block
      int S = 0;
      for (int cand = 4; cand >= 2 && !S; --cand) if (fixed + cand * tile_b <= 113 * 1024) S = cand;
      for (int cand = 4; cand >= 2 && !S; --cand) if (fixed + cand * tile_b <= 200 * 1024) S = cand;
      if (S) {
        using MmaFn = void (*)(const float*, const float*, const float*, int, const int*, int, int, int, float*, long long, int, int);
        const MmaFn fn = (S == 4) ? dec_src_attn_mma_kernel<4> : (S == 3) ? dec_src_attn_mma_kernel<3> : dec_src_attn_mma_kernel<2>;
        static bool attr[5] = {false, false, false, false, false};
        if (!attr[S]) {
          if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)) != cudaSuccess) {
            espb_set_error("dec_src_attn: cannot raise dynamic shared memory"); return ESPB_ERR_CUDA;
          }
          attr[S] = true;
        }
        espb::launch_pdl(fn, dim3(U * H), dim3(256), fixed + S * tile_b, stream, q, kmem, vmem, Tmax, lens, Wg, D, H, ctx, ctx_plane, w0, W);
        ESPB_CHECK_LAUNCH();
        continue;
      }
    }
    const size_t red = (size_t)8 * Wg * dk, scs = ((size_t)Wg * Tmax + 3) & ~(size_t)3;
    const size_t smem = ((size_t)Wg * dk + (scs > red ? scs : red) + (size_t)128 * (dk + 4)) * sizeof(float);
    if (smem > 200 * 1024) { espb_set_error("dec_src_attn: beam*T too large for shared memory"); return ESPB_ERR_ARG; }
    using KernelFn = void (*)(const float*, const float*, const float*, int, const int*, int, int, int, int, float*, long long, int, int);
    KernelFn fn = dec_src_attn_kernel<4, 0, 0>;
    if (dk == 64) {
      switch (Wg) {
        case 4: fn = dec_src_attn_kernel<4, 4, 64>; break;
        case 5: fn = dec_src_attn_kernel<4, 5, 64>; break;
        case 8: fn = dec_src_attn_kernel<4, 8, 64>; break;
        case 10: fn = dec_src_attn_kernel<4, 10, 64>; break;
        case 16: fn = dec_src_attn_kernel<4, 16, 64>; break;
        default: break;
      }
    }
    if (smem > 48 * 1024) {
      if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)) != cudaSuccess) {
        espb_set_error("dec_src_attn: cannot raise dynamic shared memory"); return ESPB_ERR_CUDA;
      }
    }
    espb::launch_pdl(fn, dim3(U * H), dim3(256), smem, stream, q, kmem, vmem, Tmax, lens, Wg, D, H, lpr, ctx, ctx_plane, w0, W);
    ESPB_CHECK_LAUNCH();
  }
  return ESPB_OK;
}

int espb_rows_topk_f32(const float* x, long long rows, long long ld, int V, float scale, int k, int* ids, float* vals, cudaStream_t stream) {
  if (k > 128 || k > V || V > 256 * 128) { espb_set_error("rows_topk: k must be <= min(128, V) and V <= 32768"); return ESPB_ERR_ARG; }
  if (V <= 256 * 4) rows_topk_kernel<4><<<(unsigned)rows, 256, 0, stream>>>(x, ld, V, scale, k, ids, vals);
  else if (V <= 256 * 20) rows_topk_kernel<20><<<(unsigned)rows, 256, 0, stream>>>(x, ld, V, scale, k, ids, vals);
  else if (V <= 256 * 40) rows_topk_kernel<40><<<(unsigned)rows, 256, 0, stream>>>(x, ld, V, scale, k, ids, vals);
  else rows_topk_kernel<128><<<(unsigned)rows, 256, 0, stream>>>(x, ld, V, scale, k, ids, vals);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_ctc_init_state_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int W, float* r, float* s_prev,
                            cudaStream_t stream) {
  const int n = U * W;
  ctc_init_state_kernel<<<(n + 63) / 64, 64, 0, stream>>>(logp, Tmax, V, lens, blank, W, n, r, s_prev);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_ctc_extend_state_f32(const float* logp, int T_new, int V, int blank, int n, const float* r_old, int T_old, float* r_new, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  if (T_old < 1 || T_new < T_old) { espb_set_error("ctc_extend_state: need 1 <= T_old <= T_new"); return ESPB_ERR_ARG; }
  ctc_extend_state_kernel<<<(n + 63) / 64, 64, 0, stream>>>(logp, T_new, V, blank, n, r_old, T_old, r_new);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_ctc_score_cands_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int eos, int W, const float* r_prev,
                             const float* s_prev, const int* last_tok, int out_len, const int* step_ptr, const int* cand, int P, float* part,
                             float* psi, int* valid, int token_major, cudaStream_t stream) {
  const int n = U * W, tot = n * (P + 1);
  ctc_score_cands_kernel<<<(tot + 7) / 8, 256, 0, stream>>>(logp, Tmax, V, lens, blank, eos, W, n, r_prev, s_prev, last_tok, out_len, step_ptr, cand,
                                                              P, part, psi, valid, token_major);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_ctc_score_dense_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int eos, int W, const float* r_prev,
                             const float* s_prev, const int* last_tok, int out_len, float* part, cudaStream_t stream) {
  const long long tot = (long long)U * W * V;
  ctc_score_dense_kernel<<<(unsigned)((tot + 127) / 128), 128, 0, stream>>>(logp, Tmax, V, lens, blank, eos, W, U * W, r_prev, s_prev, last_tok,
                                                                           out_len, part);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_beam_select(const float* score, const float* sc_dec, const float* sc_ctc, const int* active, float* n_score, float* n_sc_dec,
                     float* n_sc_ctc, int* n_active, int* n_last_tok, int* n_parent, int* bp_parent, int* bp_token, int* ended_count,
                     int* ended_step, int* ended_slot, float* ended_score, float* ended_dec, float* ended_ctc, int ended_cap, float* best_at_step,
                     float* best_all, int* utt_done, int U, int W, int P, int V, int step, const int* step_ptr, const int* maxlen,
                     const int* minlen, int eos,
                     float w_dec, float w_ctc, float penalty, int mode, const int* cand_ids, const float* cand_val, const float* logp_dec,
                     const float* part, const int* valid, int end_detect, int maxlen_cap, cudaStream_t stream) {
  const int PC = (mode == 1) ? P + 1 : P;
  if (W * PC > 256 * 28 || W > 64 || mode < 0 || mode > 2) { espb_set_error("beam_select: beam > 64, beam * candidates > 7168 or bad mode"); return ESPB_ERR_ARG; }
  BeamState st{score, sc_dec, sc_ctc, active, n_score, n_sc_dec, n_sc_ctc, n_active, n_last_tok, n_parent, bp_parent, bp_token,
               ended_count, ended_step, ended_slot, ended_score, ended_dec, ended_ctc, ended_cap, best_at_step, best_all, utt_done};
#define ESPB_BEAM_SELECT(MC, NT)                                                                                                                       \
  beam_select_kernel<MC, NT><<<U, NT, 0, stream>>>(st, U, W, P, V, step, step_ptr, maxlen, minlen, eos, w_dec, w_ctc, penalty, mode, cand_ids, cand_val, \
                                                   logp_dec, part, valid, end_detect, maxlen_cap)
  const int total = W * PC;
  if (total <= 32 * 6) ESPB_BEAM_SELECT(6, 32);
  else if (total <= 32 * 12) ESPB_BEAM_SELECT(12, 32);
  else if (total <= 32 * 24) ESPB_BEAM_SELECT(24, 32);
  else if (total <= 32 * 52 && W <= 32) ESPB_BEAM_SELECT(52, 32);
  else if (total <= 256 * 14) ESPB_BEAM_SELECT(14, 256);      // wide beams (the reference's Librispeech decode_asr.yaml: beam 60, pre-beam 90)
  else ESPB_BEAM_SELECT(28, 256);
#undef ESPB_BEAM_SELECT
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_anc_update_i32(const int* anc, int* n_anc, int anc_ld, const int* parent, int pos, const int* step_ptr, int n, cudaStream_t stream) {
  anc_update_kernel<<<n, 64, 0, stream>>>(anc, n_anc, anc_ld, parent, pos, step_ptr, n);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_ctc_advance_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int eos, int W, const float* r_prev,
                         const int* parent, const int* par_last_tok, const int* new_tok, const int* new_active, int out_len, const int* step_ptr,
                         float* r_new, float* s_new, int token_major, cudaStream_t stream) {
  const int n = U * W;
  ctc_advance_kernel<<<(n + 3) / 4, 128, 0, stream>>>(logp, Tmax, V, lens, blank, eos, W, n, r_prev, parent, par_last_tok, new_tok, new_active,
                                                       out_len, step_ptr, r_new, s_new, token_major);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_transpose_tv_f32(const float* x, int U, int Tmax, int V, float* xt, cudaStream_t stream) {
  dim3 grid((V + 31) / 32, (Tmax + 31) / 32, U), block(32, 8);
  transpose_tv_kernel<<<grid, block, 0, stream>>>(x, Tmax, V, xt);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_gather_rows_split_f32(const int* tok, const float* emb, int n, int E, float* out, long long plane, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  espb::launch_pdl(gather_rows_split_kernel, dim3(n), dim3(128), 0, stream, tok, emb, E, out, plane);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_relu_posenc_f32(float* x, int n, int D, const float* pe, int pos, const int* step_ptr, float scale, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  espb::launch_pdl(relu_posenc_kernel, dim3(n), dim3(128), 0, stream, x, D, pe, pos, step_ptr, scale);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_axpby_f32(const float* a, float wa, const float* b, float wb, float* out, long long n, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  espb::launch_pdl(axpby_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, a, wa, b, wb, out, n);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_track_scores_f32(const int* parent, const int* tok, const int* bp_parent, const float* logp_a, const float* logp_b, int V, const float* prev_a,
                          const float* prev_b, float* new_a, float* new_b, float* hist_a, float* hist_b, int step, const int* step_ptr, int n,
                          cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  track_scores_kernel<<<(n + 127) / 128, 128, 0, stream>>>(parent, tok, bp_parent, logp_a, logp_b, V, prev_a, prev_b, new_a, new_b, hist_a, hist_b, step,
                                                          step_ptr, n);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_rnnlm_gather_f32(const int* tok, const float* emb, int E, int Ep, const int* anc, int anc_ld, int pos, const int* step_ptr,
                          const float* h_ring, int L, int n, int H, int Hp, float* xs, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  if (E > Ep || H > Hp || (Ep & 3) || (Hp & 3) || L < 1) { espb_set_error("rnnlm_gather: need E <= Ep, H <= Hp, Ep and Hp multiples of 4, L >= 1"); return ESPB_ERR_ARG; }
  espb::launch_pdl(rnnlm_gather_kernel, dim3(n), dim3(128), 0, stream, tok, emb, E, Ep, anc, anc_ld, pos, step_ptr, h_ring, L, n, H, Hp, xs);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_lstm_cell_f32(const float* gates, const int* anc, int anc_ld, int pos, const int* step_ptr, float* h_ring, float* c_ring, int layer, int L,
                       int n, int H, int Hp, float* out, long long out_plane, int out_ld, cudaStream_t stream) {
  if (n <= 0) return ESPB_OK;
  if (H > Hp || layer < 0 || layer >= L || out_ld < H) { espb_set_error("lstm_cell: need H <= Hp, 0 <= layer < L, out_ld >= H"); return ESPB_ERR_ARG; }
  const long long tot = (long long)n * H;
  espb::launch_pdl(lstm_cell_kernel, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, stream, gates, anc, anc_ld, pos, step_ptr, h_ring, c_ring,
                   layer, L, n, H, Hp, out, out_plane, out_ld);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_step_inc_i32(int* step, cudaStream_t stream) {
  step_inc_kernel<<<1, 1, 0, stream>>>(step);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

int espb_count_active_i32(const int* active, int n, int* out, cudaStream_t stream) {
  count_active_kernel<<<1, 256, 0, stream>>>(active, n, out);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

}  // extern "C"
