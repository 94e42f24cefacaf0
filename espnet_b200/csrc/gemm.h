// GEMM descriptor shared by the wgmma 3xTF32 kernel and the SIMT fp32 kernel.
//
//   C[by,bx][m, n] = epilogue( sum_k A[by,bx][m, k] * B[by*bym, bx*bxm][n, k] )
//
// A and B are "split" fp32 tensors: two planes (hi, lo) `*_plane` elements apart, produced by
// espb::tf32_hi/tf32_lo; the tensor-core kernel forms A_lo*B_hi + A_hi*B_lo + A_hi*B_hi in
// fp32 register accumulators (error-compensated 3xTF32, ~2^-21 relative per product); the SIMT
// kernel adds the planes back (hi+lo is the original fp32 value up to 2^-22) and uses FFMA.
// Both operands are K-major (row-major [rows, K]).
#pragma once
#include <cuda_runtime.h>

struct EspbGemmDesc {
  int M, N, K;          // per batch slice
  int nbx, nby;         // batch grid: slice (bx, by)
  int a_mode;           // 0: general strided; 1: conv2 implicit GEMM over the parity-split conv1 output
  int kob;              // mode 0: K blocks (of 32) per "outer" A index (K = n_outer * kob * 32); <=0: none
  const float* A; long long a_plane, lda, sa_x, sa_y;   // A element (m,k): A + by*sa_y + (bx + k_outer)*sa_x + m*lda + k_inner
  const float* B; long long b_plane, ldb, sb_x, sb_y;   // sb_* may be 0 (operand shared across that batch dim)
  float* C; long long c_plane, ldc, sc_x, sc_y;
  int split_out;        // 1: write hi/lo planes (c_plane apart); 0: plain fp32
  const float* bias;    // [N] or null
  long long sbias_x;    // bias offset per batch-x index (heads as batch: bias + bx*sbias_x)
  const float* R; long long ldr, sr_x, sr_y;            // residual (may alias C) or null
  float alpha;          // out = R + alpha * act(acc + bias)   (R absent: alpha * act(...))
  int act;              // espb::ACT_*
  int cv_t1h, cv_f1h, cv_cin;  // mode 1: conv1-output half extents and channel count
  int band_t;           // > 0: only columns n with band_t-1-m <= n <= 2*band_t-2-m are ever read (rel-pos shift): tiles outside are skipped
};

int espb_gemm_tc_launch(const EspbGemmDesc& d, cudaStream_t stream, int version);  // wgmma (1: plain accumulation, 2: chunked promotion)
int espb_gemm_simt_launch(const EspbGemmDesc& d, cudaStream_t stream);  // any strides
