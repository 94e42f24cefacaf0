// Fused self-attention of the encoders on the Hopper tensor cores: S = Q K^T (+ rel-pos term) -> masked online softmax -> O = P V in one
// kernel; neither the scores nor the probabilities ever reach HBM.
//
// Reference semantics: RelPositionMultiHeadedAttention.forward / rel_shift / forward_attention
// (espnet2/legacy/nets/pytorch_backend/transformer/attention.py:416-459, 391-414, 121-151) and, with bd == nullptr, the plain
// MultiHeadedAttention.forward (:153-265): scores = (q_u k^T + bd[i][T-1-i+j]) / sqrt(d_k), keys j >= len masked, softmax, x = p v.
//
// Numerics: every product is an error-compensated 3xTF32 wgmma (a_lo b_hi + a_hi b_lo + a_hi b_hi, fp32 accumulate) like the GEMMs
// (gemm.cu).  The long accumulation over the keys does NOT run in the tensor core: every 64-key tile's P V lands in a fresh wgmma
// accumulator and is added into fp32 registers with round-to-nearest while the online-softmax rescale is applied.
//
// Work decomposition: one CTA per (utterance, head, block of 128 queries), three warpgroups.
//   warps 0-7  two consumer warpgroups; warpgroup g owns query rows [128 qb + 64 g, +64).  S = Q K^T with Q and K from shared memory,
//              + rel-pos term bd[i][T-1-i+j] read from global memory (rel_shift is a row-dependent column offset of the unshifted
//              bd = (q+v) p^T matrix), scale, mask, online softmax in registers; P hi/lo is rearranged from the accumulator layout into
//              the register A-operand layout with quad shuffles, and O(t) = P(t) V(t) reads only V^T from shared memory.
//   warp 8     TMA producer (one elected lane; its warpgroup hands its registers to the consumers): Q once, then K tiles and V^T tiles (SWIZZLE_128B, hi / lo planes) through a two-stage
//              ring each; a consumer warpgroup releases a stage once its MMAs retired.
#include <cuda.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace espb::tc;

constexpr int DK = 64;                      // head dimension served by this kernel
constexpr int KB = 64;                      // keys per tile
constexpr int QB = 128;                     // queries per CTA
constexpr int KV_STAGES = 2;
constexpr int BLK_BYTES = 64 * 128;         // one [64 rows x 32 fp32] swizzled operand block
constexpr int Q_BYTES = 2 * 2 * 2 * BLK_BYTES;          // [hi | lo] x [d_k block 0 | 1] x [row block 0 | 1]
constexpr int KV_STAGE_BYTES = 4 * BLK_BYTES;           // [hi | lo] x [k-block 0 | 1]
constexpr int ATT_THREADS = 384;          // warpgroups 0-1: consumers, warpgroup 2: producer (one warp works)

struct AttnParams {
  const float* q; long long q_plane, ldq;        // split Q-like tensor: element (row, c) of head h at q + row*ldq + h*DK + c (+ q_plane: lo)
  const int* lens;
  const float* bd; int Rp;                       // unshifted rel-pos term [B][H][T][Rp] or null
  float* out; long long out_plane, ldo;          // split context [rows][H*DK]
  int B, H, T, nqb;                              // nqb = ceil(T / 128)
  float scale;                                   // 1 / sqrt(d_k)
};

// bd values of one row for the keys key0 + 8j + 0/1, j < 8 (key0 even; row = the row's bd pointer shifted by T-1-i): pairs as one 8-byte
// load where the row's shift leaves them aligned.  Keys >= len are not read (past the band for the last key tile) and give 0.  Every
// element of v is written on every call: values kept from the previous tile would stay live across P V and spill.
__device__ __forceinline__ void load_bd_row(const float* row, int key0, int len, float2 (&v)[8]) {
  const bool vec = (reinterpret_cast<uintptr_t>(row) & 7) == 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int key = key0 + 8 * j;
    float2 x = make_float2(0.f, 0.f);
    if (row) {
      if (vec && key + 1 < len) {
        x = __ldg(reinterpret_cast<const float2*>(row + key));
      } else {
        if (key < len) x.x = __ldg(row + key);
        if (key + 1 < len) x.y = __ldg(row + key + 1);
      }
    }
    v[j] = x;
  }
}

template <bool RELPOS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
flash_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                  AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_base = smem_base;
  const uint32_t k_base = q_base + Q_BYTES;
  const uint32_t v_base = k_base + KV_STAGES * KV_STAGE_BYTES;
  const uint32_t bar_base = v_base + KV_STAGES * KV_STAGE_BYTES;
  const uint32_t q_full = bar_base, k_full = q_full + 8, k_empty = k_full + 8 * KV_STAGES, v_full = k_empty + 8 * KV_STAGES,
                 v_empty = v_full + 8 * KV_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x;
  const int qb = item % p.nqb, h = (item / p.nqb) % p.H, b = item / (p.nqb * p.H);
  const int len = min(p.lens[b], p.T);
  const int I0 = qb * QB;                      // first query row of the CTA
  const int nkt = (len + KB - 1) / KB;

  if (I0 >= len || nkt == 0) {
    // every query row of this block is padding (t >= len): defined (zero) output, no tensor work
    for (int i = threadIdx.x; i < QB * (DK / 4); i += blockDim.x) {
      const int row = I0 + i / (DK / 4), c = (i % (DK / 4)) * 4;
      if (row < p.T) {
        float* o = p.out + ((long long)b * p.T + row) * p.ldo + h * DK + c;
        *reinterpret_cast<float4*>(o) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(o + p.out_plane) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    return;
  }

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init(k_full + 8 * s, 1); mbar_init(k_empty + 8 * s, 2);   // empty: one arrival per consumer warpgroup
      mbar_init(v_full + 8 * s, 1); mbar_init(v_empty + 8 * s, 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQ) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmK) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmV) : "memory");
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================================================================== TMA producer (one elected lane)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 8 && elect_one_sync()) {
      mbar_expect_tx(q_full, Q_BYTES);
#pragma unroll
      for (int i = 0; i < 8; ++i) {   // block i = (plane, d_k block, row block)
        const int pl = i >> 2, kb = (i >> 1) & 1, rb = i & 1;
        tma_load_5d(q_base + i * BLK_BYTES, &tmQ, q_full, kb * 32, I0 + rb * 64, h, b, pl);
      }
      for (int t = 0; t < nkt; ++t) {
        const int s = t % KV_STAGES;
        const uint32_t ph = (uint32_t)((t / KV_STAGES) & 1);
        const int J0 = t * KB;
        mbar_wait(k_empty + 8 * s, ph ^ 1);
        mbar_expect_tx(k_full + 8 * s, KV_STAGE_BYTES);
#pragma unroll
        for (int i = 0; i < 4; ++i)   // block i = (plane, d_k block): 64 keys x 32 d_k
          tma_load_5d(k_base + s * KV_STAGE_BYTES + i * BLK_BYTES, &tmK, k_full + 8 * s, (i & 1) * 32, J0, h, b, i >> 1);
        mbar_wait(v_empty + 8 * s, ph ^ 1);
        mbar_expect_tx(v_full + 8 * s, KV_STAGE_BYTES);
#pragma unroll
        for (int i = 0; i < 4; ++i)   // block i = (plane, key block): 64 d_k rows x 32 keys of V^T
          tma_load_5d(v_base + s * KV_STAGE_BYTES + i * BLK_BYTES, &tmV, v_full + 8 * s, J0 + (i & 1) * 32, 0, h, b, i >> 1);
      }
    }
    return;
  }

  // ===================================================================== consumers: thread = (rows ra, ra + 8; 16 of the 64 columns)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int g = warp >> 2;
  const int ra = I0 + g * 64 + (warp & 3) * 16 + (lane >> 2), rb = ra + 8;
  const int tq = lane & 3;
  const int src0 = (lane & ~3) | (tq >> 1), src1 = src0 + 2;   // quad lanes holding P columns tq and tq + 4 of an 8-key group
  const uint32_t qa = q_base + g * BLK_BYTES;                   // this warpgroup's 64 rows of Q
  const float scale = p.scale;
  const float* bd_a = nullptr;
  const float* bd_b = nullptr;
  // rel-pos term of the keys J0 + 8j + 2tq + 0/1 of rows ra / rb: loaded at the top of the key tile, so the latency hides under the wait
  // for K and S = Q K^T (loading a whole tile ahead would keep 32 more registers live across P V, which then spills)
  float2 bdv_a[8], bdv_b[8];
  if (RELPOS) {
    const long long head = ((long long)b * p.H + h) * p.T;
    if (ra < p.T) bd_a = p.bd + (head + ra) * p.Rp + (p.T - 1 - ra);
    if (rb < p.T) bd_b = p.bd + (head + rb) * p.Rp + (p.T - 1 - rb);
  }
  float o_acc[32], ot[32], s[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) o_acc[j] = 0.f;
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  mbar_wait_spin(q_full, 0);

  for (int t = 0; t < nkt; ++t) {
    const int st = t % KV_STAGES;
    const uint32_t ph = (uint32_t)((t / KV_STAGES) & 1);
    const int J0 = t * KB;
    if (RELPOS) {
      load_bd_row(bd_a, J0 + 2 * tq, len, bdv_a);
      load_bd_row(bd_b, J0 + 2 * tq, len, bdv_b);
    }
    // ---- S = Q K^T
    mbar_wait_spin(k_full + 8 * st, ph);
    const uint32_t kt = k_base + st * KV_STAGE_BYTES;
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = 0.f;   // the first MMA ignores the old value: keeps the previous tile's registers dead
    fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DK / 8; ++kk) {
      const uint32_t off = (uint32_t)(kk >> 2) * BLK_BYTES + (uint32_t)(kk & 3) * 32;            // K: [plane][d_k block]
      const uint32_t qoff = (uint32_t)(kk >> 2) * 2 * BLK_BYTES + (uint32_t)(kk & 3) * 32;       // Q: [plane][d_k block][row block]
      const uint64_t a_hi = gmma_desc(qa + qoff), a_lo = gmma_desc(qa + 4 * BLK_BYTES + qoff);
      const uint64_t b_hi = gmma_desc(kt + off), b_lo = gmma_desc(kt + 2 * BLK_BYTES + off);
      wgmma_tf32_ss_n64(s, a_lo, b_hi, kk != 0 ? 1u : 0u);   // small terms first
      wgmma_tf32_ss_n64(s, a_hi, b_lo, 1u);
      wgmma_tf32_ss_n64(s, a_hi, b_hi, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    if ((threadIdx.x & 127) == 0) mbar_arrive_local(k_empty + 8 * st);
    // ---- + rel-pos term, mask, online softmax (rows ra: s[4j], s[4j+1]; rb: s[4j+2], s[4j+3]; key J0 + 8j + 2tq + 0/1)
    float mt_a = -INFINITY, mt_b = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = J0 + 8 * j + 2 * tq + e;
        const bool ok = key < len;
        float va = s[4 * j + e], vb = s[4 * j + 2 + e];
        if (RELPOS) {
          if (ok && bd_a) va += e ? bdv_a[j].y : bdv_a[j].x;
          if (ok && bd_b) vb += e ? bdv_b[j].y : bdv_b[j].x;
        }
        va = ok ? va : -INFINITY;
        vb = ok ? vb : -INFINITY;
        s[4 * j + e] = va; s[4 * j + 2 + e] = vb;
        mt_a = fmaxf(mt_a, va); mt_b = fmaxf(mt_b, vb);
      }
    }
    mt_a = fmaxf(mt_a, __shfl_xor_sync(0xffffffffu, mt_a, 1)); mt_a = fmaxf(mt_a, __shfl_xor_sync(0xffffffffu, mt_a, 2));
    mt_b = fmaxf(mt_b, __shfl_xor_sync(0xffffffffu, mt_b, 1)); mt_b = fmaxf(mt_b, __shfl_xor_sync(0xffffffffu, mt_b, 2));
    const float mn_a = fmaxf(m_a, mt_a * scale), mn_b = fmaxf(m_b, mt_b * scale);   // scale > 0: max commutes with the scaling
    const float al_a = __expf(m_a - mn_a), al_b = __expf(m_b - mn_b);              // first tile: exp(-inf) = 0
    float ls_a = 0.f, ls_b = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        s[4 * j + e] = __expf(fmaf(s[4 * j + e], scale, -mn_a));           // masked: exp(-inf) = 0
        s[4 * j + 2 + e] = __expf(fmaf(s[4 * j + 2 + e], scale, -mn_b));
        ls_a += s[4 * j + e]; ls_b += s[4 * j + 2 + e];
      }
    }
    l_a = fmaf(l_a, al_a, ls_a); l_b = fmaf(l_b, al_b, ls_b);
    m_a = mn_a; m_b = mn_b;
    // ---- O(t) = P(t) V(t): P from registers (accumulator layout -> A-fragment layout through quad shuffles)
    mbar_wait_spin(v_full + 8 * st, ph);
    const uint32_t vt = v_base + st * KV_STAGE_BYTES;
    uint32_t ph_hi[8][4], ph_lo[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const float x00 = __shfl_sync(0xffffffffu, s[4 * kk], src0), x01 = __shfl_sync(0xffffffffu, s[4 * kk + 1], src0);
      const float x10 = __shfl_sync(0xffffffffu, s[4 * kk], src1), x11 = __shfl_sync(0xffffffffu, s[4 * kk + 1], src1);
      const float y00 = __shfl_sync(0xffffffffu, s[4 * kk + 2], src0), y01 = __shfl_sync(0xffffffffu, s[4 * kk + 3], src0);
      const float y10 = __shfl_sync(0xffffffffu, s[4 * kk + 2], src1), y11 = __shfl_sync(0xffffffffu, s[4 * kk + 3], src1);
      const float a[4] = {(tq & 1) ? x01 : x00, (tq & 1) ? y01 : y00, (tq & 1) ? x11 : x10, (tq & 1) ? y11 : y10};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float hi = espb::tf32_hi(a[i]);
        ph_hi[kk][i] = __float_as_uint(hi);
        ph_lo[kk][i] = __float_as_uint(espb::tf32_lo(a[i], hi));
      }
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) ot[j] = 0.f;
    fence_regs(ot);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KB / 8; ++kk) {
      const uint32_t off = (uint32_t)(kk >> 2) * BLK_BYTES + (uint32_t)(kk & 3) * 32;
      const uint64_t b_hi = gmma_desc(vt + off), b_lo = gmma_desc(vt + 2 * BLK_BYTES + off);
      wgmma_tf32_rs_n64(ot, ph_lo[kk], b_hi, kk != 0 ? 1u : 0u);
      wgmma_tf32_rs_n64(ot, ph_hi[kk], b_lo, 1u);
      wgmma_tf32_rs_n64(ot, ph_hi[kk], b_hi, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(ot);
    if ((threadIdx.x & 127) == 0) mbar_arrive_local(v_empty + 8 * st);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o_acc[4 * j] = fmaf(o_acc[4 * j], al_a, ot[4 * j]); o_acc[4 * j + 1] = fmaf(o_acc[4 * j + 1], al_a, ot[4 * j + 1]);
      o_acc[4 * j + 2] = fmaf(o_acc[4 * j + 2], al_b, ot[4 * j + 2]); o_acc[4 * j + 3] = fmaf(o_acc[4 * j + 3], al_b, ot[4 * j + 3]);
    }
  }
  // ---- total row sums over the quad, normalise, store hi / lo
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1); l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1); l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r ? rb : ra;
    if (row >= p.T) continue;
    const float inv = r ? inv_b : inv_a;
    float* o = p.out + ((long long)b * p.T + row) * p.ldo + h * DK + 2 * tq;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v0 = o_acc[4 * j + 2 * r] * inv, v1 = o_acc[4 * j + 2 * r + 1] * inv;
      const float h0 = espb::tf32_hi(v0), h1 = espb::tf32_hi(v1);
      *reinterpret_cast<float2*>(o + 8 * j) = make_float2(h0, h1);
      *reinterpret_cast<float2*>(o + p.out_plane + 8 * j) = make_float2(espb::tf32_lo(v0, h0), espb::tf32_lo(v1, h1));
    }
  }
}

template <bool RELPOS>
int launch_flash(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const AttnParams& p, cudaStream_t stream) {
  constexpr int smem = Q_BYTES + 2 * KV_STAGES * KV_STAGE_BYTES + 1024 + 256;
  static_assert(smem <= 232448, "dynamic shared memory budget exceeded");
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(flash_attn_kernel<RELPOS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      espb_set_error("cudaFuncSetAttribute(max dynamic smem) failed (flash attention)");
      return ESPB_ERR_CUDA;
    }
    attr_set = true;
  }
  const long long items = (long long)p.B * p.H * p.nqb;
  flash_attn_kernel<RELPOS><<<dim3((unsigned)items), ATT_THREADS, smem, stream>>>(tmQ, tmK, tmV, p);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}

}  // namespace

extern "C" {

// Fused (rel-pos) self-attention for d_k = 64.  All tensors are device fp32.
//   q       split [2][B*T][ldq] (planes q_plane apart; first element at q + q_off): query rows (q + pos_bias_u for rel-pos attention);
//           head h at columns h*64..
//   k       split, same layout convention (k_off, k_plane, ldk): key rows;  vt split [2][B][H][64][Tp]: V transposed, keys >= len zero
//   bd      [B][H][T][Rp] unshifted (q + pos_bias_v) p^T (columns 0..2T-2), or NULL for plain attention
//   out     split [2][B*T][ldo]: context, head h at columns h*64..
int espb_flash_attn_f32(const float* q, long long q_off, long long q_plane, long long ldq, const float* k, long long k_off, long long k_plane,
                        long long ldk, const float* vt, long long vt_plane, int Tp, const float* bd, int Rp, const int* lens, int B, int H, int T,
                        int dk, float* out, long long out_plane, long long ldo, cudaStream_t stream) {
  q += q_off; k += k_off;
  if (dk != DK) { espb_set_error("flash_attn: d_k must be 64"); return ESPB_ERR_ARG; }
  if (B <= 0 || H <= 0 || T <= 0) { espb_set_error("flash_attn: bad shape"); return ESPB_ERR_ARG; }
  if ((ldq & 3) || (q_plane & 3) || (ldo & 3) || (out_plane & 3) || (reinterpret_cast<uintptr_t>(q) & 15) || (reinterpret_cast<uintptr_t>(out) & 15)) {
    espb_set_error("flash_attn: q / out must be 16-byte aligned with strides that are multiples of 4 floats");
    return ESPB_ERR_ARG;
  }
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  {
    long long dims[5] = {DK, T, H, B, 2};
    long long str[4] = {ldq, DK, (long long)T * ldq, q_plane};
    if ((rc = espb_make_tensor_map(&tmQ, q, dims, str, 32, 64, 1)) != ESPB_OK) return rc;
  }
  {
    long long dims[5] = {DK, T, H, B, 2};
    long long str[4] = {ldk, DK, (long long)T * ldk, k_plane};
    if ((rc = espb_make_tensor_map(&tmK, k, dims, str, 32, 64, 1)) != ESPB_OK) return rc;
  }
  {
    long long dims[5] = {Tp, DK, H, B, 2};
    long long str[4] = {Tp, (long long)DK * Tp, (long long)H * DK * Tp, vt_plane};
    if ((rc = espb_make_tensor_map(&tmV, vt, dims, str, 32, 64, 1)) != ESPB_OK) return rc;
  }
  AttnParams p;
  p.q = q; p.q_plane = q_plane; p.ldq = ldq; p.lens = lens; p.bd = bd; p.Rp = Rp; p.out = out; p.out_plane = out_plane; p.ldo = ldo;
  p.B = B; p.H = H; p.T = T; p.nqb = (T + QB - 1) / QB; p.scale = 1.0f / sqrtf((float)dk);
  if (bd) return launch_flash<true>(tmQ, tmK, tmV, p, stream);
  return launch_flash<false>(tmQ, tmK, tmV, p, stream);
}

}  // extern "C"
