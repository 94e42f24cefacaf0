// Error-compensated 3xTF32 GEMM on the Hopper tensor cores (wgmma tf32, fp32 accumulators in registers, operands staged by TMA
// with 128B swizzle), plus a SIMT fp32 GEMM with the same descriptor (validator for the tensor-core path and path for shapes TMA
// cannot address).
//
// The tensor-core kernel is persistent: min(tiles, SMs) CTAs, CTA c takes 128 x BN output tiles c, c + gridDim.x, ... (see tile_at for
// the order).  Warp roles per CTA (512 threads):
//   warps 0-7 : two consumer warpgroups; warpgroup g issues the wgmma for rows [64g, 64g+64) of each tile, writes the finished fp32
//               accumulators into a shared-memory staging buffer and starts the next tile's MMAs at once
//   warp 8    : TMA producer (one elected lane) -> full[s]; the consumers release a stage through empty[s] once its MMAs retired.  The
//               producer walks the CTA's tiles in the same order, so the ring runs on across tile boundaries.
//   warps 9-15: epilogue: read each staged 64 x BN half-tile, apply bias / activation / alpha / residual / hi-lo split and store it with
//               row-contiguous 16-byte accesses, while the consumers run the next tile's MMAs.
// The rel-pos band product (EspbGemmDesc::band_t > 0) has its own persistent kernel, relpos_band_kernel.
#include <cuda.h>
#include <limits.h>

#include <algorithm>
#include <cmath>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "gemm.h"
#include "tc_common.cuh"

namespace {

using namespace espb::tc;

constexpr int BM = 128;
constexpr int BK = 32;                  // 32 fp32 = 128 B = one swizzle row
constexpr int A_TILE_BYTES = BM * 128;  // one plane
constexpr int NUM_THREADS = 512;
constexpr int EPI_WARP0 = 9;            // warps 9-15 run the epilogue
constexpr int EPI_THREADS = NUM_THREADS - EPI_WARP0 * 32;
constexpr int STAGING_BYTES = 32768;    // 64 x 128 fp32 (one warpgroup's 128-column half-tile, or both warpgroups' 64-column ones)
// Registers per thread after setmaxnreg.  setmaxnreg only moves registers inside the CTA's allocation, 512 x 128 (the launch bound's
// per-thread limit), so the two consumer and two producer / epilogue warpgroups may not ask for more than 4 x 128 between them: a larger
// request never completes.  The consumers hold two 64 x BN fp32 accumulator sets; the epilogue loop needs far fewer.
constexpr int LAUNCH_REGS = (65536 / NUM_THREADS) & ~7;
constexpr int CONSUMER_REGS = 176;
constexpr int EPI_REGS = 80;
static_assert(2 * CONSUMER_REGS + 2 * EPI_REGS <= 4 * LAUNCH_REGS, "setmaxnreg split exceeds the CTA's registers");
// Chunked promotion (version 2): K is walked in chunks of CHUNK_KB k-blocks that accumulate in a fresh wgmma accumulator, which is
// then added into an fp32 register accumulator with round-to-nearest, so the long accumulation chain does not run in the tensor core.
constexpr int CHUNK_KB = 4;

// ------------------------------------------------------------------ shared epilogue
struct EpiArgs {
  float* C; long long c_plane, ldc; int split_out;
  const float* bias; const float* R; long long ldr; float alpha; int act;
};

__device__ __forceinline__ float epi_value(const EpiArgs& e, float acc, long long row, int col) {
  float v = acc;
  if (e.bias) v += __ldg(e.bias + col);
  v = espb::apply_act_acc(v, e.act);
  v *= e.alpha;
  if (e.R) v += e.R[row * e.ldr + col];
  return v;
}

// ------------------------------------------------------------------ tensor-core kernel
template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  if constexpr (BN == 128) wgmma_tf32_ss_n128(d, adesc, bdesc, accum);
  else wgmma_tf32_ss_n64(d, adesc, bdesc, accum);
}

// Tile order: batch slices outermost; within a slice the column tiles are walked in bands of `band` column tiles, and within a band the
// column tile runs fastest.  The CTAs in flight then share a few 128-row blocks of A (each read from HBM about once) and the band's B
// tiles, which the host sizes to stay in L2 next to the A stream.
struct TilePos { int m0, n0, bx, by; };

template <int BN>
__device__ __forceinline__ TilePos tile_at(const EspbGemmDesc& p, long long t, int tiles_m, int tiles_n, int band) {
  const long long per_slice = (long long)tiles_m * tiles_n;
  const int z = (int)(t / per_slice);
  int r = (int)(t - z * per_slice);
  const int band_tiles = tiles_m * band;
  const int b = r / band_tiles;
  r -= b * band_tiles;
  const int w = min(band, tiles_n - b * band);   // the last band may be narrower
  TilePos tp;
  tp.m0 = (r / w) * BM; tp.n0 = (b * band + r % w) * BN; tp.bx = z % p.nbx; tp.by = z / p.nbx;
  return tp;
}

// Four columns col..col + 3 of a row of a bias or residual operand; columns past N read as 0.  vec: ptr + col is 16-byte aligned.
__device__ __forceinline__ float4 ld_quad(const float* ptr, int col, int N, bool vec) {
  if (vec && col + 3 < N) return *reinterpret_cast<const float4*>(ptr + col);
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = col + i < N ? ptr[col + i] : 0.f;
  return make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ float4 ldg_quad(const float* ptr, int col, int N, bool vec) {
  if (vec && col + 3 < N) return __ldg(reinterpret_cast<const float4*>(ptr + col));
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = col + i < N ? __ldg(ptr + col + i) : 0.f;
  return make_float4(v[0], v[1], v[2], v[3]);
}

// epi_value with the bias and residual values already loaded.
__device__ __forceinline__ float epi_apply(const EpiArgs& e, float acc, float b, float r) {
  float v = acc;
  if (e.bias) v += b;
  v = espb::apply_act_acc(v, e.act);
  v *= e.alpha;
  if (e.R) v += r;
  return v;
}

// Stores four horizontally adjacent epilogue values (row, col..col + 3).  vec: 16-byte stores are aligned (ldc, c_plane, the slice
// offset and C itself); otherwise, and at the last columns of a ragged N, element by element.
__device__ __forceinline__ void epi_store4(const EpiArgs& e, int row, int col, const float (&t)[4], int N, bool vec) {
  float* crow = e.C + (long long)row * e.ldc;
  if (vec && col + 3 < N) {
    if (e.split_out) {
      float h[4], l[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { h[i] = espb::tf32_hi(t[i]); l[i] = espb::tf32_lo(t[i], h[i]); }
      *reinterpret_cast<float4*>(crow + col) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(crow + e.c_plane + col) = make_float4(l[0], l[1], l[2], l[3]);
    } else {
      *reinterpret_cast<float4*>(crow + col) = make_float4(t[0], t[1], t[2], t[3]);
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (col + i >= N) break;
    if (e.split_out) { const float h = espb::tf32_hi(t[i]); crow[col + i] = h; crow[e.c_plane + col + i] = espb::tf32_lo(t[i], h); }
    else crow[col + i] = t[i];
  }
}

// Staging buffer of one 64 x BN half-tile: row r at r * BN floats, its 16-byte chunk q at chunk q ^ 2 (r & 3).  The consumers' 8-byte
// fragment stores (a half-warp writes two chunks of each of 4 consecutive rows) and the epilogue's row-contiguous 16-byte loads are
// then both free of bank conflicts.
template <int BN>
__device__ __forceinline__ uint32_t staging_off(int r, int c) {
  return (uint32_t)(r * BN + ((((c >> 2) ^ ((r & 3) << 1))) << 2) + (c & 3)) * 4u;
}

// One warpgroup's finished 64 x BN accumulators (fragment layout, tc_common.cuh) into the staging buffer at buf.
template <int BN>
__device__ __forceinline__ void stage_tile(uint32_t buf, const float (&d)[BN / 2], int r0, int c0) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(buf + staging_off<BN>(r0 + 8 * h, c0 + 8 * j)), "f"(d[4 * j + 2 * h]),
                   "f"(d[4 * j + 2 * h + 1])
                   : "memory");
}

__device__ __forceinline__ float4 ld_shared_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}

// Epilogue warps: every tile of this CTA, its two 64-row halves in order.  A thread owns four columns of the tile (the bias values are
// loaded once per tile) and a row every RPP rows; the residual loads of EPI_U such rows are issued before the first of them is stored.  R is
// either C itself (each element read and then written by the same thread) or disjoint from C (gemm.h), so no store can feed a load.
constexpr int EPI_U = 4;

template <int BN>
__device__ __forceinline__ void epilogue_warps(const EspbGemmDesc& p, long long ntiles, int tiles_m, int tiles_n, int band, uint32_t staging,
                                               uint32_t stg_full, uint32_t stg_empty) {
  constexpr int NBUF = STAGING_BYTES / (64 * BN * 4);   // 1: the warpgroups take turns on one buffer; 2: one buffer each
  constexpr int TPR = BN / 4, RPP = EPI_THREADS / TPR;  // threads per row, rows per pass
  const int et = threadIdx.x - EPI_WARP0 * 32;
  const int r_first = et / TPR, cc = 4 * (et % TPR);
  int it = 0;   // this CTA's tile ordinal: selects the staging barriers' phase
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    const TilePos tp = tile_at<BN>(p, t, tiles_m, tiles_n, band);
    EpiArgs e;
    const long long coff = (long long)tp.by * p.sc_y + (long long)tp.bx * p.sc_x;
    const long long roff = (long long)tp.by * p.sr_y + (long long)tp.bx * p.sr_x;
    e.C = p.C + coff; e.c_plane = p.c_plane; e.ldc = p.ldc; e.split_out = p.split_out;
    e.bias = p.bias ? p.bias + (long long)tp.bx * p.sbias_x : nullptr; e.R = p.R ? p.R + roff : nullptr;
    e.ldr = p.ldr; e.alpha = p.alpha; e.act = p.act;
    const bool c_vec = ((p.ldc & 3) == 0) && ((coff & 3) == 0) && ((p.c_plane & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);
    const bool r_vec = ((p.ldr & 3) == 0) && ((reinterpret_cast<uintptr_t>(e.R) & 15) == 0);
    const int col = tp.n0 + cc;
    const float4 bv = e.bias ? ldg_quad(e.bias, col, p.N, (reinterpret_cast<uintptr_t>(e.bias) & 15) == 0) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int g = 0; g < 2; ++g) {
      mbar_wait(stg_full + 8 * g, (uint32_t)it & 1);
      const uint32_t buf = staging + (NBUF == 1 ? 0 : g) * (64 * BN * 4);
      const int row_base = tp.m0 + 64 * g;
#pragma unroll 1
      for (int r0 = r_first; r0 < 64; r0 += EPI_U * RPP) {
        float4 rv[EPI_U];
#pragma unroll
        for (int u = 0; u < EPI_U; ++u) {
          const int r = r0 + u * RPP, row = row_base + r;
          rv[u] = (e.R && r < 64 && row < p.M) ? ld_quad(e.R + (long long)row * e.ldr, col, p.N, r_vec) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < EPI_U; ++u) {
          const int r = r0 + u * RPP, row = row_base + r;
          if (r >= 64 || row >= p.M) break;
          const float4 a = ld_shared_f4(buf + staging_off<BN>(r, cc));
          const float v[4] = {epi_apply(e, a.x, bv.x, rv[u].x), epi_apply(e, a.y, bv.y, rv[u].y), epi_apply(e, a.z, bv.z, rv[u].z),
                              epi_apply(e, a.w, bv.w, rv[u].w)};
          epi_store4(e, row, col, v, p.N, c_vec);
        }
      }
      mbar_arrive_local(stg_empty + 8 * (NBUF == 1 ? g ^ 1 : g));   // with one buffer, half g's release lets the other warpgroup write
    }
  }
}

template <int BN, int STAGES, bool PROMOTE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, EspbGemmDesc p, int bxm, int bym, int axm, int aym,
                   int tiles_m, int tiles_n, int band) {
  constexpr int B_TILE_BYTES = BN * 128;
  constexpr int STAGE_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
  constexpr int NR = BN / 2;   // accumulator registers per thread: a 64 x BN warpgroup tile over 128 threads
  constexpr int NBUF = STAGING_BYTES / (64 * BN * 4);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t staging = smem_base + STAGES * STAGE_BYTES;
  const uint32_t full_bar = staging + STAGING_BYTES, empty_bar = full_bar + 8 * STAGES;
  const uint32_t stg_full = empty_bar + 8 * STAGES, stg_empty = stg_full + 16;   // per consumer warpgroup

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = (p.K + BK - 1) / BK;
  const long long ntiles = (long long)tiles_m * tiles_n * p.nbx * p.nby;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 2); }   // empty: one arrival per consumer warpgroup
    for (int g = 0; g < 2; ++g) { mbar_init(stg_full + 8 * g, 128); mbar_init(stg_empty + 8 * g, EPI_THREADS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();
  espb::pdl_trigger();   // barriers and descriptors are ready: the next kernel may start its own setup
  espb::pdl_wait();      // first global access (TMA loads of A / B) follows

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(EPI_REGS));
    if (warp >= EPI_WARP0) {
      epilogue_warps<BN>(p, ntiles, tiles_m, tiles_n, band, staging, stg_full, stg_empty);
      return;
    }
    if (elect_one_sync()) {   // one lane, known to ptxas: uniform-datapath issue without per-instruction waterfall loops
      const int cblk = (p.a_mode != 0) ? p.cv_cin / BK : 0;
      const ConvGeom g = conv_geom(p.a_mode);
      int s = 0;
      uint32_t ph = 0;
      for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const TilePos tp = tile_at<BN>(p, t, tiles_m, tiles_n, band);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar + 8 * s, ph ^ 1);
          const uint32_t fb = full_bar + 8 * s;
          mbar_expect_tx(fb, STAGE_BYTES);
          const uint32_t sa = smem_base + s * STAGE_BYTES;
          if (p.a_mode == 0) {
            const int ko = (p.kob > 0) ? kb / p.kob : 0;
            const int ki = (p.kob > 0) ? kb % p.kob : kb;
            tma_load_5d(sa, &tmA, fb, ki * BK, tp.m0, tp.bx * axm + ko, tp.by * aym, 0);
            tma_load_5d(sa + A_TILE_BYTES, &tmA, fb, ki * BK, tp.m0, tp.bx * axm + ko, tp.by * aym, 1);
          } else {  // conv: tap (kt,kf) of the k x k / stride-s window over the phase-split input (conv_geom)
            const int tap = kb / cblk, c0 = (kb % cblk) * BK;
            const int kt = tap / g.k, kf = tap - kt * g.k;
            const int par = (kt % g.s) * g.s + kf % g.s;
            tma_load_5d(sa, &tmA, fb, c0, tp.m0 + kt / g.s, tp.bx + kf / g.s, par, tp.by);
            tma_load_5d(sa + A_TILE_BYTES, &tmA, fb, c0, tp.m0 + kt / g.s, tp.bx + kf / g.s, g.s * g.s + par, tp.by);
          }
          tma_load_5d(sa + 2 * A_TILE_BYTES, &tmB, fb, kb * BK, tp.n0, tp.bx * bxm, tp.by * bym, 0);
          tma_load_5d(sa + 2 * A_TILE_BYTES + B_TILE_BYTES, &tmB, fb, kb * BK, tp.n0, tp.bx * bxm, tp.by * bym, 1);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int row_in_half = (warp & 3) * 16 + (lane >> 2), col_in_tile = 2 * (lane & 3);
  const uint32_t my_buf = staging + (NBUF == 1 ? 0 : wg) * (64 * BN * 4);
  // With one staging buffer warpgroup 1 writes after the epilogue read warpgroup 0's half of the same tile: its first wait blocks.
  const uint32_t stg_parity0 = (NBUF == 1 && wg == 1) ? 0u : 1u;
  int s = 0;
  uint32_t ph = 0;
  float acc[NR], part[NR];
  int it = 0;   // this CTA's tile ordinal
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    // part is overwritten by the first MMA (scale-d 0); zeroing it here keeps it dead, not live in registers, across the handoff
#pragma unroll
    for (int i = 0; i < NR; ++i) { acc[i] = 0.f; part[i] = 0.f; }
    // Each k-block's MMAs retire before its stage is released.  Keeping one k-block in flight (wait_group 1) would hold a second stage
    // per consumer and leave the producer one k-block of lead in the 3-stage ring that fits at BN = 128; measured on H100 that was
    // slower for long K (conv2: 86 vs 72 ms) and no faster elsewhere.
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar + 8 * s, ph);   // measured: spinning here gained nothing on the encoder shapes and cost 3 % at M640 N512 K2048
      const uint32_t sa = smem_base + s * STAGE_BYTES + wg * 64 * 128;   // this warpgroup's 64 rows of A (8 KB: swizzle atoms stay aligned)
      const uint32_t sb = smem_base + s * STAGE_BYTES + 2 * A_TILE_BYTES;
      const bool fresh = PROMOTE ? (kb % CHUNK_KB == 0) : (kb == 0);
      fence_regs(part);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 8; ++k) {   // 8 tf32 = 32 bytes per MMA
        const uint64_t a_hi = gmma_desc(sa + k * 32), a_lo = gmma_desc(sa + A_TILE_BYTES + k * 32);
        const uint64_t b_hi = gmma_desc(sb + k * 32), b_lo = gmma_desc(sb + B_TILE_BYTES + k * 32);
        wgmma_tf32<BN>(part, a_lo, b_hi, (fresh && k == 0) ? 0u : 1u);   // small terms first
        wgmma_tf32<BN>(part, a_hi, b_lo, 1u);
        wgmma_tf32<BN>(part, a_hi, b_hi, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(part);
      if (wg_leader) mbar_arrive_local(empty_bar + 8 * s);   // this warpgroup no longer reads the stage
      if (PROMOTE && (kb % CHUNK_KB == CHUNK_KB - 1 || kb == num_kb - 1)) {
#pragma unroll
        for (int i = 0; i < NR; ++i) acc[i] += part[i];
      }
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    // hand the tile to the epilogue warps and go on with the next one
    mbar_wait(stg_empty + 8 * wg, ((uint32_t)it & 1) ^ stg_parity0);
    stage_tile<BN>(my_buf, PROMOTE ? acc : part, row_in_half, col_in_tile);
    mbar_arrive_local(stg_full + 8 * wg);
  }
}

// ------------------------------------------------------------------ rel-pos band kernel (EspbGemmDesc::band_t > 0)
// Row m of the band product needs only columns [T-1-m, 2T-2-m] (T = band_t).  A work unit is one (batch slice, 128-row block): its
// rows of A (hi / lo, all of K <= 128) are loaded once, and the B tiles over the columns the block reaches, [T-1-m_last, 2T-2-m0]
// (about T + 127 columns), stream through a TMA ring of k-block slots.  The grid is persistent (CTA c takes units c, c + gridDim.x, ...)
// and each consumer warpgroup keeps two accumulator sets, so the MMAs of column tile n+1 run while the stores of tile n drain.  Only
// in-band elements are stored.  Per output element the MMA sequence is the generic kernel's (per k8 step a_lo b_hi, a_hi b_lo, a_hi b_hi,
// one fp32 chain over K <= 128 = one promotion chunk), so the stored values are bit-identical to it.
constexpr int BAND_MAX_KB = 4;        // K <= 128
constexpr int BAND_SMEM = 232448;     // dynamic shared memory of the band kernel (the sm_90 maximum)
constexpr int BAND_THREADS = 384;     // warpgroups 0-1: consumers (two accumulator sets each), warpgroup 2: producer (one warp works)

struct BandTile {
  int k;        // round-robin ordinal of the work unit within this CTA (unit blockIdx.x + k * gridDim.x); -1: no more work
  int seq;      // units with tiles this CTA processed before this one: selects the A buffer and its barrier phase (units without
                // in-band columns are skipped and do not count)
  int t, nt;    // column tile within the unit, tiles of the unit
  int m0, n0;   // first row and first column of the tile
  int bx, by;   // batch slice
};

// The first unit of this CTA at ordinal >= k that has in-band columns, at its tile 0; seq units with tiles came before it.
__device__ __forceinline__ void band_unit(const EspbGemmDesc& p, int nmb, int k, int seq, int bn, BandTile& w) {
  const long long nunits = (long long)nmb * p.nbx * p.nby;
  for (;; ++k) {
    const long long u = blockIdx.x + (long long)k * gridDim.x;
    if (u >= nunits) { w.k = -1; return; }
    const int mb = (int)(u % nmb), z = (int)(u / nmb);
    const int m0 = mb * BM, mlast = min(p.M, m0 + BM) - 1;
    const int lo = max(0, p.band_t - 1 - mlast), hi = min(p.N - 1, 2 * p.band_t - 2 - m0);
    if (hi < lo) continue;
    const int n_start = lo & ~7;   // 32-byte aligned columns: the 8 consecutive floats a quad stores fill one sector
    w.k = k; w.seq = seq; w.t = 0; w.nt = (hi - n_start) / bn + 1; w.m0 = m0; w.n0 = n_start; w.bx = z % p.nbx; w.by = z / p.nbx;
    return;
  }
}
__device__ __forceinline__ void band_next(const EspbGemmDesc& p, int nmb, int bn, BandTile& w) {
  if (w.t + 1 < w.nt) { ++w.t; w.n0 += bn; return; }
  band_unit(p, nmb, w.k + 1, w.seq + 1, bn, w);
}

__device__ __forceinline__ void st_global_v2_if(float* ptr, float a, float b, bool pred) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p st.global.v2.f32 [%0], {%1, %2};\n\t}" ::"l"(ptr), "f"(a), "f"(b), "r"((int)pred)
               : "memory");
}
__device__ __forceinline__ void st_global_if(float* ptr, float a, bool pred) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.global.f32 [%0], %1;\n\t}" ::"l"(ptr), "f"(a), "r"((int)pred) : "memory");
}

// Shared memory: [nabuf A buffers of num_kb x (hi | lo) x 128 rows][stages B slots of (hi | lo) x BN rows][barriers].  With two A
// buffers the next unit's rows load while the current unit runs; with one, they load once the unit's last MMAs retired.
// NKB = ceil(K / 32) k-blocks; 128-column tiles keep A and a ring of at least NKB slots in shared memory up to NKB = 3, beyond that the
// tiles are 64 columns wide.
template <int NKB>
constexpr int band_bn() { return NKB <= 3 ? 128 : 64; }

template <int NKB, bool PROMOTE>
__global__ void __launch_bounds__(BAND_THREADS, 1)
relpos_band_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, EspbGemmDesc p, int bxm, int bym, int axm,
                   int aym, int nabuf, int stages) {
  constexpr int BN = band_bn<NKB>();
  constexpr int SLOT_BYTES = 2 * BN * 128;   // one k-block of B, hi | lo
  constexpr int NR = BN / 2;
  constexpr int num_kb = NKB;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_bytes = (uint32_t)num_kb * 2 * A_TILE_BYTES;
  const uint32_t ring = smem_base + nabuf * a_bytes;
  const uint32_t full_bar = ring + stages * SLOT_BYTES, empty_bar = full_bar + 8 * stages;
  const uint32_t a_full = empty_bar + 8 * stages, a_empty = a_full + 16;
  const int nmb = (p.M + BM - 1) / BM;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 2); }
    for (int i = 0; i < 2; ++i) { mbar_init(a_full + 8 * i, 1); mbar_init(a_empty + 8 * i, 2); }   // empty: one arrival per consumer warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();
  espb::pdl_trigger();
  espb::pdl_wait();

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");   // the producer warpgroup hands its registers to the consumers
    if (warp == 8 && elect_one_sync()) {
      int s = 0;
      uint32_t ph = 0;
      BandTile w;
      for (band_unit(p, nmb, 0, 0, BN, w); w.k >= 0; band_next(p, nmb, BN, w)) {
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar + 8 * s, ph ^ 1);
          const uint32_t fb = full_bar + 8 * s, sb = ring + s * SLOT_BYTES;
          mbar_expect_tx(fb, SLOT_BYTES);
          tma_load_5d(sb, &tmB, fb, kb * BK, w.n0, w.bx * bxm, w.by * bym, 0);
          tma_load_5d(sb + BN * 128, &tmB, fb, kb * BK, w.n0, w.bx * bxm, w.by * bym, 1);
          if (++s == stages) { s = 0; ph ^= 1; }
        }
        if (w.t == 0) {   // after the unit's first B tile: with one A buffer this waits until the previous unit's MMAs retired
          const int ab = w.seq % nabuf;
          mbar_wait(a_empty + 8 * ab, ((uint32_t)(w.seq / nabuf) & 1) ^ 1);
          const uint32_t fa = a_full + 8 * ab, sa = smem_base + ab * a_bytes;
          mbar_expect_tx(fa, a_bytes);
          for (int kb = 0; kb < num_kb; ++kb) {
            const int ko = (p.kob > 0) ? kb / p.kob : 0;
            const int ki = (p.kob > 0) ? kb % p.kob : kb;
            tma_load_5d(sa + kb * 2 * A_TILE_BYTES, &tmA, fa, ki * BK, w.m0, w.bx * axm + ko, w.by * aym, 0);
            tma_load_5d(sa + kb * 2 * A_TILE_BYTES + A_TILE_BYTES, &tmA, fa, ki * BK, w.m0, w.bx * axm + ko, w.by * aym, 1);
          }
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  int s = 0, rs = 0;   // ring slot of the next acquire / release
  uint32_t ph = 0;
  // MMAs of tile w into d (asynchronous: committed, not waited for)
  auto issue = [&](const BandTile& w, float (&d)[NR]) {
    const int ab = w.seq % nabuf;
    if (w.t == 0) mbar_wait_spin(a_full + 8 * ab, (uint32_t)(w.seq / nabuf) & 1);
    const uint32_t sa = smem_base + ab * a_bytes + wg * 64 * 128;   // this warpgroup's 64 rows of A
    // every slot of the tile is waited for before the first MMA: no barrier-wait loop runs while MMAs are in flight
    uint32_t sb[num_kb];
#pragma unroll
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait_spin(full_bar + 8 * s, ph);
      sb[kb] = ring + s * SLOT_BYTES;
      if (++s == stages) { s = 0; ph ^= 1; }
    }
    fence_regs(d);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < num_kb; ++kb) {
      const uint32_t sak = sa + kb * 2 * A_TILE_BYTES;
#pragma unroll
      for (int k = 0; k < BK / 8; ++k) {
        const uint64_t a_hi = gmma_desc(sak + k * 32), a_lo = gmma_desc(sak + A_TILE_BYTES + k * 32);
        const uint64_t b_hi = gmma_desc(sb[kb] + k * 32), b_lo = gmma_desc(sb[kb] + BN * 128 + k * 32);
        wgmma_tf32<BN>(d, a_lo, b_hi, (kb == 0 && k == 0) ? 0u : 1u);   // small terms first
        wgmma_tf32<BN>(d, a_hi, b_lo, 1u);
        wgmma_tf32<BN>(d, a_hi, b_hi, 1u);
      }
    }
    wgmma_commit();
  };
  // After the MMAs of w retired: hand its B slots (and, after the unit's last tile, its A buffer) back to the producer.
  auto release = [&](const BandTile& w) {
    for (int kb = 0; kb < num_kb; ++kb) {
      if (wg_leader) mbar_arrive_local(empty_bar + 8 * rs);
      if (++rs == stages) rs = 0;
    }
    if (w.t == w.nt - 1 && wg_leader) mbar_arrive_local(a_empty + 8 * (w.seq % nabuf));
  };
  // Plain epilogue (alpha * acc) of the in-band elements.  Branch-free (predicated stores): the next tile's MMAs are in flight meanwhile,
  // and ptxas serialises wgmma whose accumulators stay live across divergent control flow.
  const bool vec_ok = ((p.ldc & 1) == 0) && ((p.sc_x & 1) == 0) && ((p.sc_y & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
  auto store = [&](const BandTile& w, const float (&d)[NR]) {
    float* const cbase = p.C + (long long)w.by * p.sc_y + (long long)w.bx * p.sc_x;
    const int row0 = w.m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int col = w.n0 + 2 * (lane & 3);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = row0 + 8 * r;
      float* const crow = cbase + (long long)row * p.ldc;
      // in-band columns [lo, end); none for rows past M
      const int lo = p.band_t - 1 - row, end = row < p.M ? min(p.N, 2 * p.band_t - 1 - row) : INT_MIN;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = col + 8 * j;
        float v0 = d[4 * j + 2 * r], v1 = d[4 * j + 2 * r + 1];
        if (PROMOTE) { v0 = 0.f + v0; v1 = 0.f + v1; }   // the generic kernel's promotion of its single chunk into a zeroed accumulator
        v0 *= p.alpha; v1 *= p.alpha;
        const bool in0 = c >= lo && c < end, in1 = c + 1 >= lo && c + 1 < end;
        const bool pair = vec_ok && in0 && in1;
        st_global_v2_if(crow + c, v0, v1, pair);
        st_global_if(crow + c, v0, in0 && !pair);
        st_global_if(crow + c + 1, v1, in1 && !pair);
      }
    }
  };
  // Tile cur's MMAs are in flight in dc: retire them, start the next tile's MMAs in dn and store cur while they run.  Returns false after
  // the last tile.  Between the issue into dn and the wait at the top of the next step the code is straight-line.
  auto step = [&](BandTile& cur, float (&dc)[NR], float (&dn)[NR]) -> bool {
    wgmma_wait<0>();
    fence_regs(dc);
    BandTile nxt = cur;
    band_next(p, nmb, BN, nxt);
    release(cur);
    if (nxt.k < 0) { store(cur, dc); return false; }
    issue(nxt, dn);
    store(cur, dc);
    cur = nxt;
    return true;
  };

  float acc0[NR], acc1[NR];
  BandTile cur;
  band_unit(p, nmb, 0, 0, BN, cur);
  if (cur.k < 0) return;
  issue(cur, acc0);
  for (;;) {
    if (!step(cur, acc0, acc1)) break;
    if (!step(cur, acc1, acc0)) break;
  }
}

// ------------------------------------------------------------------ SIMT kernel (fp32 FFMA)
__device__ __forceinline__ float load_a(const EspbGemmDesc& p, int bx, int by, int m, int k) {
  if (m >= p.M || k >= p.K) return 0.f;
  long long off;
  if (p.a_mode == 0) {
    int ko = 0, ki = k;
    if (p.kob > 0) { ko = k / (p.kob * BK); ki = k % (p.kob * BK); }
    off = (long long)by * p.sa_y + (long long)(bx + ko) * p.sa_x + (long long)m * p.lda + ki;
    return p.A[off] + p.A[off + p.a_plane];
  }
  // conv over [b][plane*s*s + pt*s + pf][F_in/s][T_in/s][C] (conv_geom)
  const ConvGeom g = conv_geom(p.a_mode);
  const int tap = k / p.cv_cin, c = k % p.cv_cin, kt = tap / g.k, kf = tap % g.k;
  const int par = (kt % g.s) * g.s + kf % g.s, nph = g.s * g.s;
  const int tt = m + kt / g.s, ff = bx + kf / g.s;
  if (tt >= p.cv_t1h || ff >= p.cv_f1h) return 0.f;
  const long long sub = (long long)p.cv_f1h * p.cv_t1h * p.cv_cin;
  off = (long long)by * 2 * nph * sub + ((long long)ff * p.cv_t1h + tt) * p.cv_cin + c;
  return p.A[off + par * sub] + p.A[off + (nph + par) * sub];
}
__device__ __forceinline__ float load_b(const EspbGemmDesc& p, int bx, int by, int n, int k) {
  if (n >= p.N || k >= p.K) return 0.f;
  long long off = (long long)by * p.sb_y + (long long)bx * p.sb_x + (long long)n * p.ldb + k;
  return p.B[off] + p.B[off + p.b_plane];
}

__global__ void __launch_bounds__(256) gemm_simt_kernel(EspbGemmDesc p) {
  __shared__ float As[16][65], Bs[16][65];
  const int bx = blockIdx.z % p.nbx, by = blockIdx.z / p.nbx;
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  if (p.band_t > 0 && ((n0 + 63 < p.band_t - 1 - (m0 + 63)) || (n0 > 2 * p.band_t - 2 - m0))) return;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < p.K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      int r = i >> 4, kk = i & 15;
      As[kk][r] = load_a(p, bx, by, m0 + r, k0 + kk);
      Bs[kk][r] = load_b(p, bx, by, n0 + r, k0 + kk);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  EpiArgs e;
  e.C = p.C + (long long)by * p.sc_y + (long long)bx * p.sc_x; e.c_plane = p.c_plane; e.ldc = p.ldc; e.split_out = p.split_out;
  e.bias = p.bias ? p.bias + (long long)bx * p.sbias_x : nullptr; e.R = p.R ? p.R + (long long)by * p.sr_y + (long long)bx * p.sr_x : nullptr;
  e.ldr = p.ldr; e.alpha = p.alpha; e.act = p.act;
  for (int i = 0; i < 4; ++i) {
    const int row = m0 + ty * 4 + i;
    if (row >= p.M) continue;
    for (int j = 0; j < 4; ++j) {
      const int col = n0 + tx * 4 + j;
      if (col >= p.N) continue;
      float t = epi_value(e, acc[i][j], row, col);
      float* c = e.C + (long long)row * e.ldc + col;
      if (e.split_out) { float h = espb::tf32_hi(t); c[0] = h; c[e.c_plane] = espb::tf32_lo(t, h); }
      else c[0] = t;
    }
  }
}

// ------------------------------------------------------------------ host side
int make_map(CUtensorMap* map, const float* base, const long long dims[5], const long long strides_el[4], int box_rows) {
  return espb_make_tensor_map(map, base, dims, strides_el, BK, box_rows, 1);
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 1;
  }
  return n;
}

// B (hi and lo planes) up to GEMM_B_L2_BYTES stays in L2 across the waves of an unbanded walk; larger B is walked in bands of up to
// GEMM_B_BAND_BYTES.  Measured on H100 (50 MB L2), M = 59968: the CTC head (N 5000, K 512: B = 20 MB) ran 3.25-3.30 ms unbanded against
// 4.14-4.20 ms in 8 MiB bands; the Transformer's FFN w1 (N 4096, K 1024: B = 32 MB) ran 6.09-6.13 ms in 8 MiB bands against 6.57-6.74
// unbanded, and 6.28-6.31 ms with 4, 8 or 16 MiB bands.  The threshold lies between those two B sizes.  (The 3.25-3.30 ms CTC head was
// measured with spinning consumers; with the current waits it runs 4.27-4.47 ms unbanded, as banded: the threshold is neutral there.)
constexpr long long GEMM_B_L2_BYTES = 24ll << 20;
constexpr long long GEMM_B_BAND_BYTES = 8ll << 20;

// Column tiles per band (tile_at).  Estimated HBM bytes per batch slice: one band over all columns reads A once, and B once if B stays
// in L2, else once per wave of SM-count tiles (the CTAs of a wave that share a column tile share its reads).  Narrower bands read A
// once per band and keep their B in L2.  Bands are used only where that estimate is lower: they pay off for wide B over many row blocks
// (the Transformer's FFN w1 and CTC head), not where a few row blocks have a long K (conv2, embed.out: A is read per band).
int column_band(const EspbGemmDesc& d, int bn, int tiles_m, int tiles_n) {
  const double a_bytes = 2.0 * tiles_m * BM * d.K * sizeof(float), tile_b = 2.0 * bn * d.K * sizeof(float), b_bytes = tiles_n * tile_b;
  if (b_bytes <= GEMM_B_L2_BYTES) return tiles_n;
  const int w = (int)std::max(1.0, std::floor(GEMM_B_BAND_BYTES / tile_b));
  if (w >= tiles_n) return tiles_n;
  const double waves_per_b = tiles_m / std::max(1.0, (double)num_sms() / tiles_n);
  const double whole = a_bytes + b_bytes * waves_per_b, banded = a_bytes * ((tiles_n + w - 1) / w) + b_bytes;
  return banded < whole ? w : tiles_n;
}

template <int BN, int STAGES, bool PROMOTE>
int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const EspbGemmDesc& d, int bxm, int bym, int axm, int aym, cudaStream_t stream) {
  constexpr int smem = STAGES * (2 * A_TILE_BYTES + 2 * BN * 128) + STAGING_BYTES + 1024 + 16 * STAGES + 32;
  static_assert(smem <= 232448, "dynamic shared memory budget exceeded");
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_tf32x3_kernel<BN, STAGES, PROMOTE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      espb_set_error("cudaFuncSetAttribute(max dynamic smem) failed");
      return ESPB_ERR_CUDA;
    }
    attr_set = true;
  }
  const int tiles_m = (d.M + BM - 1) / BM, tiles_n = (d.N + BN - 1) / BN;
  const int band = column_band(d, BN, tiles_m, tiles_n);
  const long long tiles = (long long)tiles_m * tiles_n * d.nbx * d.nby;
  const int grid = (int)std::min(tiles, (long long)num_sms());
  if (espb::launch_pdl(gemm_tf32x3_kernel<BN, STAGES, PROMOTE>, dim3(grid), dim3(NUM_THREADS), smem, stream, tmA, tmB, d, bxm, bym, axm, aym, tiles_m,
                       tiles_n, band) != cudaSuccess) {
    espb_set_error(cudaGetErrorString(cudaGetLastError())); return ESPB_ERR_CUDA;
  }
  return ESPB_OK;
}

// Lowest and highest byte address of the elements (m, n) of a strided [M, N] window over nbx x nby slices.
void window_span(const float* base, long long ld, long long sx, long long sy, const EspbGemmDesc& d, uintptr_t& lo, uintptr_t& hi) {
  long long a = 0, b = (long long)(d.M - 1) * ld + (d.N - 1);
  const long long ex = (long long)(d.nbx - 1) * sx, ey = (long long)(d.nby - 1) * sy;
  (ex < 0 ? a : b) += ex;
  (ey < 0 ? a : b) += ey;
  lo = reinterpret_cast<uintptr_t>(base + a);
  hi = reinterpret_cast<uintptr_t>(base + b) + sizeof(float) - 1;
}

// The epilogue contract of gemm.h: R is C itself or shares no address range with what the GEMM writes.
bool residual_ok(const EspbGemmDesc& d) {
  if (!d.R) return true;
  if (d.R == d.C && d.ldr == d.ldc && d.sr_x == d.sc_x && d.sr_y == d.sc_y) return true;
  uintptr_t rlo, rhi, clo, chi;
  window_span(d.R, d.ldr, d.sr_x, d.sr_y, d, rlo, rhi);
  for (int plane = 0; plane < (d.split_out ? 2 : 1); ++plane) {
    window_span(d.C + plane * d.c_plane, d.ldc, d.sc_x, d.sc_y, d, clo, chi);
    if (rlo <= chi && clo <= rhi) return false;
  }
  return true;
}

template <int NKB, bool PROMOTE>
int launch_band(const CUtensorMap& tmA, const CUtensorMap& tmB, const EspbGemmDesc& d, int bxm, int bym, int axm, int aym, cudaStream_t stream) {
  constexpr int BN = band_bn<NKB>();
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(relpos_band_kernel<NKB, PROMOTE>, cudaFuncAttributeMaxDynamicSharedMemorySize, BAND_SMEM) != cudaSuccess) {
      espb_set_error("cudaFuncSetAttribute(max dynamic smem) failed (band GEMM)");
      return ESPB_ERR_CUDA;
    }
    attr_set = true;
  }
  const int num_kb = NKB;
  const int a_bytes = num_kb * 2 * A_TILE_BYTES, slot = 2 * BN * 128;
  const int budget = BAND_SMEM - 1024 - 256;   // alignment slack, barriers
  const int nabuf = (2 * a_bytes + (num_kb + 1) * slot <= budget) ? 2 : 1;
  const int stages = min(8, (budget - nabuf * a_bytes) / slot);
  if (stages < num_kb) { espb_set_error("band GEMM: K too large for the shared-memory ring"); return ESPB_ERR_ARG; }
  const long long units = (long long)((d.M + BM - 1) / BM) * d.nbx * d.nby;
  const int grid = (int)(units < num_sms() ? units : num_sms());
  const int smem = 1024 + nabuf * a_bytes + stages * slot + 16 * stages + 32;
  if (espb::launch_pdl(relpos_band_kernel<NKB, PROMOTE>, dim3(grid), dim3(BAND_THREADS), smem, stream, tmA, tmB, d, bxm, bym, axm, aym, nabuf,
                       stages) != cudaSuccess) {
    espb_set_error(cudaGetErrorString(cudaGetLastError())); return ESPB_ERR_CUDA;
  }
  return ESPB_OK;
}
}  // namespace

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn espb_get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// 5-D fp32 tensor map, 128B swizzle, box = {32, box_rows, 1, 1, 1}. strides in elements for dims 1..4.
int espb_make_tensor_map(CUtensorMap* map, const float* base, const long long dims[5], const long long strides_el[4], int box0, int box1,
                         int swizzle128) {
  EncodeTiledFn fn = espb_get_encode_fn();
  if (!fn) { espb_set_error("cuTensorMapEncodeTiled entry point not available"); return ESPB_ERR_TMA; }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t box[5] = {(cuuint32_t)box0, (cuuint32_t)box1, 1, 1, 1}, estr[5] = {1, 1, 1, 1, 1};
  long long packed = 1;
  for (int i = 0; i < 5; ++i) {
    gdim[i] = (cuuint64_t)(dims[i] > 0 ? dims[i] : 1);
  }
  packed = (long long)gdim[0];
  for (int i = 0; i < 4; ++i) {
    long long s = strides_el[i];
    if (s <= 0) s = ((packed + 3) / 4) * 4;  // unused / broadcast dim (size 1): any legal stride
    if (s % 4 != 0) { espb_set_error("TMA stride not a multiple of 16 bytes"); return ESPB_ERR_TMA; }
    gstr[i] = (cuuint64_t)s * 4ull;
    packed = s * (long long)gdim[i + 1];
  }
  if (reinterpret_cast<uintptr_t>(base) & 15) { espb_set_error("TMA base not 16-byte aligned"); return ESPB_ERR_TMA; }
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d) dims=[%lld,%lld,%lld,%lld,%lld] strides=[%lld,%lld,%lld,%lld]", (int)r,
             dims[0], dims[1], dims[2], dims[3], dims[4], strides_el[0], strides_el[1], strides_el[2], strides_el[3]);
    espb_set_error(buf);
    return ESPB_ERR_TMA;
  }
  return ESPB_OK;
}


int espb_gemm_tc_launch(const EspbGemmDesc& d, cudaStream_t stream, int version) {
  if (d.M <= 0 || d.N <= 0 || d.K <= 0 || d.nbx <= 0 || d.nby <= 0) { espb_set_error("gemm: bad shape"); return ESPB_ERR_ARG; }
  if (!residual_ok(d)) { espb_set_error("gemm: residual R partially overlaps the output C"); return ESPB_ERR_ARG; }
  CUtensorMap tmA, tmB;
  int rc;
  int axm = 1, aym = 1;
  if (d.a_mode == 0) {
    long long n_outer = 1, k_inner = d.K;
    if (d.kob > 0) { k_inner = (long long)d.kob * BK; n_outer = (d.K + k_inner - 1) / k_inner; }
    axm = (d.sa_x != 0 && d.nbx > 1) ? 1 : 0;   // operand shared across a batch dim -> coordinate 0
    aym = (d.sa_y != 0 && d.nby > 1) ? 1 : 0;
    long long dims[5] = {k_inner, d.M, (axm ? d.nbx : 1) + n_outer - 1, aym ? d.nby : 1, 2};
    long long str[4] = {d.lda, d.sa_x, d.sa_y, d.a_plane};
    rc = make_map(&tmA, d.A, dims, str, BM);
  } else {
    const ConvGeom g = conv_geom(d.a_mode);
    if (d.cv_cin % BK != 0 || d.K != g.k * g.k * d.cv_cin) {
      espb_set_error("conv gemm: cin must be a multiple of 32 and K = k*k*cin");
      return ESPB_ERR_ARG;
    }
    const long long sub = (long long)d.cv_f1h * d.cv_t1h * d.cv_cin, nph = g.s * g.s;
    long long dims[5] = {d.cv_cin, d.cv_t1h, d.cv_f1h, 2 * nph, d.nby};
    long long str[4] = {d.cv_cin, (long long)d.cv_t1h * d.cv_cin, sub, 2 * nph * sub};
    rc = make_map(&tmA, d.A, dims, str, BM);
  }
  if (rc != ESPB_OK) return rc;
  const int bxm = d.sb_x != 0 ? 1 : 0, bym = d.sb_y != 0 ? 1 : 0;
  // rel-pos band product: the band kernel takes a strided A operand, K <= 128 and the plain epilogue (alpha only); any other band
  // descriptor runs through the generic kernel below, which computes every element (a superset of the band)
  if (d.band_t > 0 && d.a_mode == 0 && d.K <= BAND_MAX_KB * BK && !d.bias && !d.R && d.act == espb::ACT_NONE && !d.split_out) {
    const int nkb = (d.K + BK - 1) / BK;
    long long dims[5] = {d.K, d.N, bxm ? d.nbx : 1, bym ? d.nby : 1, 2};
    long long str[4] = {d.ldb, d.sb_x, d.sb_y, d.b_plane};
    if ((rc = make_map(&tmB, d.B, dims, str, nkb <= 3 ? band_bn<3>() : band_bn<4>())) != ESPB_OK) return rc;
    const bool pr = version == 2;
    switch (nkb) {
      case 1: return pr ? launch_band<1, true>(tmA, tmB, d, bxm, bym, axm, aym, stream) : launch_band<1, false>(tmA, tmB, d, bxm, bym, axm, aym, stream);
      case 2: return pr ? launch_band<2, true>(tmA, tmB, d, bxm, bym, axm, aym, stream) : launch_band<2, false>(tmA, tmB, d, bxm, bym, axm, aym, stream);
      case 3: return pr ? launch_band<3, true>(tmA, tmB, d, bxm, bym, axm, aym, stream) : launch_band<3, false>(tmA, tmB, d, bxm, bym, axm, aym, stream);
      default: return pr ? launch_band<4, true>(tmA, tmB, d, bxm, bym, axm, aym, stream) : launch_band<4, false>(tmA, tmB, d, bxm, bym, axm, aym, stream);
    }
  }
  const long long tiles_m = (d.M + BM - 1) / BM, nb = (long long)d.nbx * d.nby;
  // 128-column tiles unless the problem then has fewer tiles than SMs (decode-step shapes): 64-column tiles spread it over more SMs
  const int bn = (d.N <= 64 || tiles_m * ((d.N + 127) / 128) * nb < num_sms()) ? 64 : 128;
  {
    long long dims[5] = {d.K, d.N, bxm ? d.nbx : 1, bym ? d.nby : 1, 2};
    long long str[4] = {d.ldb, d.sb_x, d.sb_y, d.b_plane};
    rc = make_map(&tmB, d.B, dims, str, bn);
    if (rc != ESPB_OK) return rc;
  }
  if (version == 2) {
    if (bn == 128) return launch_tc<128, 3, true>(tmA, tmB, d, bxm, bym, axm, aym, stream);
    return launch_tc<64, 4, true>(tmA, tmB, d, bxm, bym, axm, aym, stream);
  }
  if (bn == 128) return launch_tc<128, 3, false>(tmA, tmB, d, bxm, bym, axm, aym, stream);
  return launch_tc<64, 4, false>(tmA, tmB, d, bxm, bym, axm, aym, stream);
}

int espb_gemm_simt_launch(const EspbGemmDesc& d, cudaStream_t stream) {
  if (d.M <= 0 || d.N <= 0 || d.K <= 0 || d.nbx <= 0 || d.nby <= 0) { espb_set_error("gemm: bad shape"); return ESPB_ERR_ARG; }
  if (!residual_ok(d)) { espb_set_error("gemm: residual R partially overlaps the output C"); return ESPB_ERR_ARG; }
  dim3 grid((d.M + 63) / 64, (d.N + 63) / 64, d.nbx * d.nby);
  gemm_simt_kernel<<<grid, 256, 0, stream>>>(d);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}
