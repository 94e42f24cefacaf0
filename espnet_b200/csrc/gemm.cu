// Error-compensated 3xTF32 GEMM on the Hopper tensor cores (wgmma tf32, fp32 accumulators in registers, operands staged by TMA
// with 128B swizzle), plus a SIMT fp32 GEMM with the same descriptor (validator for the tensor-core path and path for shapes TMA
// cannot address).
//
// Warp roles per CTA (288 threads, one 128 x BN output tile):
//   warps 0-7: two consumer warpgroups; warpgroup g issues the wgmma for rows [64g, 64g+64) of the tile and runs their epilogue
//              (bias / activation / residual / hi-lo split) straight from the accumulator registers
//   warp 8   : TMA producer (one elected lane) -> full[s]; the consumers release a stage through empty[s] once its MMAs retired
#include <cuda.h>
#include <limits.h>
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
constexpr int NUM_THREADS = 288;
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
// rel-pos band (EspbGemmDesc::band_t): a tile of rows [m0, m0+bm) x columns [n0, n0+bn) is needed iff it intersects
// { (m, n) : T-1-m <= n <= 2T-2-m }.
__device__ __forceinline__ bool band_skip(int T, int m0, int bm, int n0, int bn) {
  if (T <= 0) return false;
  return (n0 + bn - 1 < T - 1 - (m0 + bm - 1)) || (n0 > 2 * T - 2 - m0);
}

template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  if constexpr (BN == 128) wgmma_tf32_ss_n128(d, adesc, bdesc, accum);
  else wgmma_tf32_ss_n64(d, adesc, bdesc, accum);
}

// Epilogue of two horizontally adjacent accumulator elements (row, col) and (row, col + 1).
__device__ __forceinline__ void epi_store2(const EpiArgs& e, int row, int col, float v0, float v1, int M, int N, bool vec_ok) {
  if (row >= M || col >= N) return;
  float* crow = e.C + (long long)row * e.ldc;
  const bool two = col + 1 < N;
  const float t0 = epi_value(e, v0, row, col), t1 = two ? epi_value(e, v1, row, col + 1) : 0.f;
  if (vec_ok && two) {
    if (e.split_out) {
      const float h0 = espb::tf32_hi(t0), h1 = espb::tf32_hi(t1);
      *reinterpret_cast<float2*>(crow + col) = make_float2(h0, h1);
      *reinterpret_cast<float2*>(crow + e.c_plane + col) = make_float2(espb::tf32_lo(t0, h0), espb::tf32_lo(t1, h1));
    } else {
      *reinterpret_cast<float2*>(crow + col) = make_float2(t0, t1);
    }
    return;
  }
  const float t[2] = {t0, t1};
  for (int i = 0; i < (two ? 2 : 1); ++i) {
    if (e.split_out) { const float h = espb::tf32_hi(t[i]); crow[col + i] = h; crow[e.c_plane + col + i] = espb::tf32_lo(t[i], h); }
    else crow[col + i] = t[i];
  }
}

template <int BN, int STAGES, bool PROMOTE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, EspbGemmDesc p, int bxm, int bym, int axm, int aym) {
  constexpr int B_TILE_BYTES = BN * 128;
  constexpr int STAGE_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
  constexpr int NR = BN / 2;   // accumulator registers per thread: a 64 x BN warpgroup tile over 128 threads
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full_bar = smem_base + STAGES * STAGE_BYTES, empty_bar = full_bar + 8 * STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int bx = blockIdx.z % p.nbx, by = blockIdx.z / p.nbx;
  const int num_kb = (p.K + BK - 1) / BK;
  if (band_skip(p.band_t, m0, BM, n0, BN)) {   // tile outside the rel-pos band
    espb::pdl_wait();
    return;
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 2); }   // empty: one arrival per consumer warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();
  espb::pdl_trigger();   // barriers and descriptors are ready: the next kernel may start its own setup
  espb::pdl_wait();      // first global access (TMA loads of A / B) follows

  if (warp == 8) {
    if (elect_one_sync()) {   // one lane, known to ptxas: uniform-datapath issue without per-instruction waterfall loops
      const int cblk = (p.a_mode == 1) ? p.cv_cin / BK : 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(empty_bar + 8 * s, ph ^ 1);
        const uint32_t fb = full_bar + 8 * s;
        mbar_expect_tx(fb, STAGE_BYTES);
        const uint32_t sa = smem_base + s * STAGE_BYTES;
        if (p.a_mode == 0) {
          const int ko = (p.kob > 0) ? kb / p.kob : 0;
          const int ki = (p.kob > 0) ? kb % p.kob : kb;
          tma_load_5d(sa, &tmA, fb, ki * BK, m0, bx * axm + ko, by * aym, 0);
          tma_load_5d(sa + A_TILE_BYTES, &tmA, fb, ki * BK, m0, bx * axm + ko, by * aym, 1);
        } else {  // conv2: tap (kt,kf) of the 3x3/stride-2 window over the parity-split conv1 output
          const int tap = kb / cblk, c0 = (kb % cblk) * BK;
          const int kt = tap / 3, kf = tap % 3;
          const int par = (kt & 1) * 2 + (kf & 1);
          tma_load_5d(sa, &tmA, fb, c0, m0 + (kt >> 1), bx + (kf >> 1), par, by);
          tma_load_5d(sa + A_TILE_BYTES, &tmA, fb, c0, m0 + (kt >> 1), bx + (kf >> 1), 4 + par, by);
        }
        tma_load_5d(sa + 2 * A_TILE_BYTES, &tmB, fb, kb * BK, n0, bx * bxm, by * bym, 0);
        tma_load_5d(sa + 2 * A_TILE_BYTES + B_TILE_BYTES, &tmB, fb, kb * BK, n0, bx * bxm, by * bym, 1);
      }
    }
    return;
  }

  const int wg = warp >> 2;
  float acc[NR], part[NR];
#pragma unroll
  for (int i = 0; i < NR; ++i) { acc[i] = 0.f; part[i] = 0.f; }
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(full_bar + 8 * s, (kb / STAGES) & 1);
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
    if ((threadIdx.x & 127) == 0) mbar_arrive_local(empty_bar + 8 * s);   // this warpgroup no longer reads the stage
    if (PROMOTE && (kb % CHUNK_KB == CHUNK_KB - 1 || kb == num_kb - 1)) {
#pragma unroll
      for (int i = 0; i < NR; ++i) acc[i] += part[i];
    }
  }

  EpiArgs e;
  const long long coff = (long long)by * p.sc_y + (long long)bx * p.sc_x;
  const long long roff = (long long)by * p.sr_y + (long long)bx * p.sr_x;
  e.C = p.C + coff; e.c_plane = p.c_plane; e.ldc = p.ldc; e.split_out = p.split_out;
  e.bias = p.bias ? p.bias + (long long)bx * p.sbias_x : nullptr; e.R = p.R ? p.R + roff : nullptr;
  e.ldr = p.ldr; e.alpha = p.alpha; e.act = p.act;
  const bool vec_ok = ((p.ldc & 1) == 0) && ((coff & 1) == 0) && ((p.c_plane & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
  const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int col = n0 + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const float* r = PROMOTE ? acc : part;
    epi_store2(e, row, col + 8 * j, r[4 * j], r[4 * j + 1], p.M, p.N, vec_ok);
    epi_store2(e, row + 8, col + 8 * j, r[4 * j + 2], r[4 * j + 3], p.M, p.N, vec_ok);
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
  // conv2 over [b][plane*4 + pt*2 + pf][F1h][T1h][C]
  const int tap = k / p.cv_cin, c = k % p.cv_cin, kt = tap / 3, kf = tap % 3;
  const int par = (kt & 1) * 2 + (kf & 1);
  const int tt = m + (kt >> 1), ff = bx + (kf >> 1);
  if (tt >= p.cv_t1h || ff >= p.cv_f1h) return 0.f;
  const long long sub = (long long)p.cv_f1h * p.cv_t1h * p.cv_cin;
  off = (long long)by * 8 * sub + ((long long)ff * p.cv_t1h + tt) * p.cv_cin + c;
  return p.A[off + par * sub] + p.A[off + (4 + par) * sub];
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

template <int BN, int STAGES, bool PROMOTE>
int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const EspbGemmDesc& d, int bxm, int bym, int axm, int aym, cudaStream_t stream) {
  constexpr int smem = STAGES * (2 * A_TILE_BYTES + 2 * BN * 128) + 1024 + 16 * STAGES;
  static_assert(smem <= 232448, "dynamic shared memory budget exceeded");
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_tf32x3_kernel<BN, STAGES, PROMOTE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      espb_set_error("cudaFuncSetAttribute(max dynamic smem) failed");
      return ESPB_ERR_CUDA;
    }
    attr_set = true;
  }
  dim3 grid((d.M + BM - 1) / BM, (d.N + BN - 1) / BN, d.nbx * d.nby);
  if (espb::launch_pdl(gemm_tf32x3_kernel<BN, STAGES, PROMOTE>, grid, dim3(NUM_THREADS), smem, stream, tmA, tmB, d, bxm, bym, axm, aym) != cudaSuccess) {
    espb_set_error(cudaGetErrorString(cudaGetLastError())); return ESPB_ERR_CUDA;
  }
  return ESPB_OK;
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
    if (d.cv_cin % BK != 0 || d.K != 9 * d.cv_cin) { espb_set_error("conv2 gemm: cin must be a multiple of 32"); return ESPB_ERR_ARG; }
    const long long sub = (long long)d.cv_f1h * d.cv_t1h * d.cv_cin;
    long long dims[5] = {d.cv_cin, d.cv_t1h, d.cv_f1h, 8, d.nby};
    long long str[4] = {d.cv_cin, (long long)d.cv_t1h * d.cv_cin, sub, 8 * sub};
    rc = make_map(&tmA, d.A, dims, str, BM);
  }
  if (rc != ESPB_OK) return rc;
  const int bxm = d.sb_x != 0 ? 1 : 0, bym = d.sb_y != 0 ? 1 : 0;
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
  dim3 grid((d.M + 63) / 64, (d.N + 63) / 64, d.nbx * d.nby);
  gemm_simt_kernel<<<grid, 256, 0, stream>>>(d);
  ESPB_CHECK_LAUNCH();
  return ESPB_OK;
}
