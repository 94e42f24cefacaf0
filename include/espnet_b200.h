/* espnet_b200.h -- C ABI of libespnet_b200.so (H100 / sm_90a kernels for ESPnet2's Speech2Text path).
 *
 * The reference has no FFI for this path: its boundary is Python classes + registries + state_dict
 * (SURVEY.md 8b).  Each entry point below replaces the ATen call sequence of one reference function and is
 * what a reference-side binding (ctypes, see INTEGRATION.md) would call.  Conventions:
 *   - every function returns 0 on success, a negative code on failure (espb_last_error() has the text);
 *   - all pointers are DEVICE pointers unless stated; no allocation, no ownership transfer, caller provides
 *     workspaces; everything is enqueued on `stream` and returns immediately;
 *   - float tensors are fp32; "split" tensors are two fp32 planes (tf32 hi, lo) `plane` elements apart that
 *     feed the tensor-core GEMM (EspbGemmDesc);
 *   - lengths: `long long` where the reference uses int64 tensors (waveform / feature lengths), `int` for
 *     encoder-frame lengths and token ids produced by this library.
 */
#ifndef ESPNET_B200_H
#define ESPNET_B200_H

#include <cuda_runtime.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ESPB_ACT_NONE 0
#define ESPB_ACT_RELU 1
#define ESPB_ACT_SWISH 2
#define ESPB_ACT_GELU 3

const char* espb_last_error(void);
int espb_abi_version(void);
int espb_device_sm(int* major, int* minor);

/* ---- GEMM: every nn.Linear / 1x1 Conv1d / Conv2d(C,C,k,s) / batched attention matmul on the path --------------
 * C[by,bx] = R + alpha * act(A[by,bx] (M x K) * B[by,bx]^T (N x K) + bias), operands split (hi/lo planes).
 * Replaces torch.matmul / F.linear at: positionwise_feed_forward.py:30-32, attention.py:77-119,146,448-452,
 * convolution.py:66,77 (pointwise convs), subsampling.py:400-406,451,606-611,711-716,818-825 (convs as implicit GEMM a_mode 1..3, embed.out
 * with kob), ctc.py:39 (ctc_lo), transformer_decoder.py:227-234 (output_layer), decoder_layer.py (all Linears).
 * use_tc=1: wgmma tf32, 3 MMAs per product (A_lo*B_hi + A_hi*B_lo + A_hi*B_hi), TMA operands
 *           (needs 16-byte aligned bases/strides); use_tc=0: SIMT fp32 FFMA kernel, any strides. */
typedef struct EspbGemmDesc {
  int M, N, K;
  int nbx, nby;
  int a_mode;          /* 0 general; 1..3 implicit-GEMM Conv2d(C, C, k, s) over an input split into its s*s phases
                          [b][plane*s*s + (t%s)*s + (f%s)][cv_f1h][cv_t1h][C] (espb_conv1_relu_phase_f32, espb_phase_split_f32):
                          row m = output time, batch x = output frequency, K = k*k*C ordered (kt, kf, c), nby = batch;
                          1: k 3, s 2 (subsampling.py:400-406 Conv2dSubsampling; Conv2dSubsampling8 :818-825, both strided convs);
                          2: k 3, s 1 (Conv2dSubsampling2, subsampling.py:606-611);
                          3: k 5, s 3 (Conv2dSubsampling6, subsampling.py:711-716) */
  int kob;             /* mode 0: K blocks (32) per outer A index; <=0 none */
  const float* A; long long a_plane, lda, sa_x, sa_y;
  const float* B; long long b_plane, ldb, sb_x, sb_y;
  float* C; long long c_plane, ldc, sc_x, sc_y;
  int split_out;
  const float* bias; long long sbias_x;   /* bias + bx*sbias_x */
  const float* R; long long ldr, sr_x, sr_y;
  float alpha;
  int act;
  int cv_t1h, cv_f1h, cv_cin;   /* a_mode 1..3: ceil(T_in/s), ceil(F_in/s) of the conv input, its channel count (a multiple of 32) */
  int band_t;          /* > 0: rel-pos band -- only elements of row m in columns [band_t-1-m, 2*band_t-2-m] are defined in C afterwards
                          (the band kernel serves a_mode 0, K <= 128 and the plain epilogue; other descriptors compute all of C) */
} EspbGemmDesc;
int espb_gemm_f32(const EspbGemmDesc* d, int use_tc, cudaStream_t stream);

/* ---- Frontend: Stft.forward + power + LogMel.forward in one kernel ----------------------------------------------
 * espnet2/layers/stft.py:75-120 (torch.stft n_fft 512, any hop <= 1024, center/reflect, any window, onesided),
 * espnet2/asr/frontend/default.py:110 (re^2+im^2), espnet2/layers/log_mel.py:57-84 (matmul melmat, clamp 1e-10, log,
 * zero padded frames).  wave [B][Lmax] (utterance b's samples at wave + b*Lmax; samples >= len are not read), out
 * [B][Tf_max][n_mels], Tf = 1 + len/hop frames per utterance, frames Tf..Tf_max-1 set to 0.  The mel matrix is passed in the
 * sparse form (start/count/offset per filter + packed weights); tw512[k] = (cos, -sin)(2 pi k / 512), k < 256.
 * partial [B][espb_frontend_blocks(Tf_max)][n_mels] receives per-block column sums (32 frames per block, frames >= Tf not
 * counted) for the MVN kernel (may be NULL). */
int espb_frontend_blocks(int Tf_max);
/* hop: 1..1024 (Tf = 1 + len/hop); window: 512 taps (a shorter win_length is zero-padded around the centre by the caller, as torch.stft
 * does); tw256t[k1*16 + n2] = (cos, -sin)(2 pi n2 k1 / 256), the twiddles of the 16 x 16 four-step FFT; mel_nnz = number of packed weights
 * (<= 4096); n_mels <= 128.  Refused with ESPB_ERR_ARG otherwise.  Preconditions the kernel does not check: every length > 256 (the
 * reflect padding of 256 samples needs them), Tf_max >= 1 + max len / hop, and partial (if not NULL) sized
 * [B][espb_frontend_blocks(Tf_max)][n_mels]. */
int espb_stft_logmel_f32(const float* wave, const long long* wave_lens, int B, int Lmax, int hop, const float* window, const float* tw512,
                         const float* tw256t, const int* mel_start, const int* mel_count, const int* mel_offset, const float* mel_weight,
                         int mel_nnz, int n_mels, float* out, int Tf_max, float* partial, cudaStream_t stream);
/* UtteranceMVN.forward, norm_means only (espnet2/layers/utterance_mvn.py:45-88), in place, n_mels <= 128.  _from_partial takes the
 * partial sums espb_stft_logmel_f32 wrote for these features (Tf = 1 + wave_len/hop); espb_utt_mvn_f32 computes its own into partial_ws
 * [B][(Tf_max + 31)/32][n_mels].  Rows t < len get x - mean over those rows; rows t >= len are neither read nor written (the reference
 * would set them to -mean in a zero-padded batch; every consumer here ignores them). */
int espb_utt_mvn_from_partial_f32(float* feats, const long long* wave_lens, int B, int Tf_max, int n_mels, int hop, const float* partial,
                                  cudaStream_t stream);
int espb_utt_mvn_f32(float* feats, const long long* feat_lens, int B, int Tf_max, int n_mels, float* partial_ws, cudaStream_t stream);
/* GlobalMVN.forward (espnet2/layers/global_mvn.py:74-103), in place: (x - mean) masked to the valid frames, then / std. */
int espb_global_mvn_f32(float* feats, const long long* feat_lens, int B, int Tmax, int D, const float* mean, const float* stdv, int norm_means,
                        int norm_vars, cudaStream_t stream);

/* ---- Encoder glue kernels -----------------------------------------------------------------------------------
 * LayerNorm (transformer/layer_norm.py:12-42, eps 1e-12): out_plain and/or out_split may be NULL. */
int espb_layernorm_f32(const float* x, long long rows, int D, const float* gamma, const float* beta, float eps, float* out_plain,
                       float* out_split, long long split_plane, cudaStream_t stream);
/* fp32 -> tf32 hi/lo planes (weights, positional table). */
int espb_split_tf32_f32(const float* x, long long n, float* out, long long plane, cudaStream_t stream);
/* Conv2d(1,C,3,2)+ReLU (subsampling.py:400-402): feats [B][Tf_max][F] -> [B][8][F1h][T1h][C] parity-split planes
 * (espb_conv1_relu_phase_f32 with s = 2). */
int espb_conv1_relu_f32(const float* feats, int B, int Tf_max, int F, const float* w, const float* bias, int C, float* out, int T1, int F1,
                        int T1h, int F1h, cudaStream_t stream);
/* The first Conv2d(1,C,3,2)+ReLU of Conv2dSubsampling2/6/8 (subsampling.py:606-611,711-716,818-825) with its output split into the s*s
 * phases of the next conv's stride s in 1..3: [B][plane*s*s + (t1%s)*s + (f1%s)][F1h][T1h][C], F1h = ceil(F1/s), T1h = ceil(T1/s). */
int espb_conv1_relu_phase_f32(const float* feats, int B, int Tf_max, int F, const float* w, const float* bias, int C, float* out, int T1, int F1,
                              int s, int T1h, int F1h, cudaStream_t stream);
/* Conv2dSubsampling8's second conv output -> input of its third (subsampling.py:818-825): x split [B][F][T][C] (planes x_plane apart) ->
 * [B][plane*s*s + (t%s)*s + (f%s)][Fh][Th][C] with Fh = ceil(F/s), Th = ceil(T/s); C, x_plane multiples of 4, x / out 16-byte aligned. */
int espb_phase_split_f32(const float* x, long long x_plane, int B, int F, int T, int C, int s, int Th, int Fh, float* out, cudaStream_t stream);
/* q + pos_bias_u / q + pos_bias_v (attention.py:441-444) from the split qkv buffer [M][3D]. */
int espb_qu_qv_f32(const float* qkv, long long qkv_plane, long long M, int D, const float* pos_u, const float* pos_v, float* qu, float* qv,
                   long long out_plane, cudaStream_t stream);
/* v.transpose for the P*V GEMM: [b][t][h*dk+d] -> split [b][h][dk][Tp], rows t >= lens[b] zeroed. */
int espb_v_transpose_f32(const float* qkv, long long qkv_plane, int B, int Tmax, int D, int H, const int* lens, float* vt,
                         long long vt_plane, int Tp, cudaStream_t stream);
/* rel_shift + /sqrt(d_k) + key mask + softmax (attention.py:391-414,455-457,121-151): ac [B][H][T][Tp], bd [B][H][T][Rp]. */
int espb_relpos_softmax_f32(const float* ac, const float* bd, int B, int H, int T, int Tp, int Rp, const int* lens, float sqrt_dk,
                            float* probs, long long probs_plane, cudaStream_t stream);
/* MultiHeadedAttention default branch (attention.py:121-151,262-265; TransformerEncoder, SURVEY 8f-1): probs = softmax(scores / sqrt_dk) over the
 * keys j < lens[b], 0 elsewhere; scores [B][H][T][Tp] -> probs hi/lo planes [B][H][T][Tp]. */
int espb_masked_softmax_f32(const float* scores, int B, int H, int T, int Tp, const int* lens, float sqrt_dk, float* probs, long long probs_plane,
                            cudaStream_t stream);
/* Fused self-attention for d_k = 64 on wgmma (attention.py:416-459 rel-pos, :153-265 plain; scores and probabilities never reach HBM):
 * out[b,i,h,:] = softmax_j<len_b( (q[b,i,h,:] . k[b,j,h,:] + bd[b,h,i,T-1-i+j]) / sqrt(d_k) ) . v[b,j,h,:].
 * q / k / out are split (hi/lo plane) tensors (first element at q + q_off / k + k_off) with row strides ldq / ldk / ldo, head h at columns h*64..; vt is the split V^T [B][H][64][Tp]
 * written by espb_v_transpose_f32; bd is the UNSHIFTED (q + pos_bias_v) p^T product [B][H][T][Rp] (rel_shift is applied while loading) or NULL
 * for absolute-position attention.  Replaces the q k^T GEMM + espb_relpos_softmax_f32 / espb_masked_softmax_f32 + p v GEMM sequence.
 * vt must hold zeros at keys >= len (espb_v_transpose_f32 writes them): those keys get weight 0, and 0 * NaN would not be 0.  Only keys
 * < len of k and only the band columns T-1-i .. T-1-i+len-1 of bd row i are read.  An utterance with len = 0 gets an all-zero output, as
 * does every 128-query block that starts at or beyond len; query rows len <= t < T of a block that also holds valid rows are finite.
 * d_k must be 64, B, H, T > 0; ldq, q_plane, ldo, out_plane multiples of 4 and q, out 16-byte aligned; ldk, k_plane, vt_plane and
 * Tp multiples of 4 (TMA strides).  Refused with ESPB_ERR_ARG / ESPB_ERR_TMA otherwise. */
int espb_flash_attn_f32(const float* q, long long q_off, long long q_plane, long long ldq, const float* k, long long k_off, long long k_plane,
                        long long ldk, const float* vt, long long vt_plane, int Tp, const float* bd, int Rp, const int* lens, int B, int H, int T,
                        int dk, float* out, long long out_plane, long long ldo, cudaStream_t stream);
/* GLU -> depthwise Conv1d(K, pad (K-1)/2) -> BatchNorm1d(eval, folded) -> Swish (conformer/convolution.py:56-79). */
int espb_glu_dwconv_bn_swish_f32(const float* y, int B, int Tmax, int C, const int* lens, const float* dw_w, const float* dw_b, int K,
                                 const float* bn_a, const float* bn_b, float* out, long long out_plane, cudaStream_t stream);
int espb_zero_pad_rows_f32(float* x, int B, int Tmax, int D, const int* lens, long long plane, int nplanes, cudaStream_t stream);
/* E-Branchformer cgMLP gating unit, identity gate (espnet2/asr/layers/cgmlp.py:57-81): h [B][Tmax][U] (channel_proj1 + GELU output, plain)
 * -> out[b][t][c] = h[..][c] * (dwconv_K(LayerNorm_eps(h[..][U/2 ..]))[t][c] + conv_b[c]) as split [B*Tmax][U/2], U/2 <= 2048.  The conv sees
 * zeros outside [0, lens[b]); rows t >= lens[b] of out are 0.  stats: caller workspace of 2 * B * Tmax floats (per-row mean / rstd); the
 * normalised gate itself is never written to memory.  conv_w [U/2][K], K odd <= 127. */
int espb_csgu_f32(const float* h, int B, int Tmax, int U, const int* lens, const float* ln_g, const float* ln_b, float eps, const float* conv_w,
                  const float* conv_b, int K, float* stats, float* out, long long out_plane, cudaStream_t stream);
/* E-Branchformer merge (e_branchformer_encoder.py:166-170): cat [B][Tmax][C2] plain -> out = split(cat + dwconv_K(cat) + b) [B*Tmax][C2],
 * depthwise over C2 channels with zeros outside [0, lens[b]); rows t >= lens[b] of out are 0.  w [C2][K], K odd <= 127. */
int espb_merge_dwconv_f32(const float* cat, int B, int Tmax, int C2, const int* lens, const float* w, const float* b, int K, float* out,
                          long long out_plane, cudaStream_t stream);
/* Branchformer learned_ave merge weights (branchformer_encoder.py:221-266): x1 / x2 [B][Tmax] rows of D floats at row stride ldx (plain).
 * For branch k of utterance b, over its rows t < lens[b] only: s_t = (x_t . pool_w[k] + pool_b[k]) / sqrt(D), p = softmax_t(s),
 * weight_k = (sum_t p_t x_t) . weight_w[k] + weight_b[k]; merge_w[b][0..1] = softmax(weight_0, weight_1).  pool_w / weight_w [2][D],
 * pool_b / weight_b [2].  One read of the rows (online softmax over 32-row chunks, then a combine launch); no host synchronisation.
 * part: caller workspace of B * 2 * ceil(Tmax / 32) * (D + 2) floats. */
int espb_branch_pool_f32(const float* x1, const float* x2, long long ldx, int B, int Tmax, int D, const int* lens, const float* pool_w,
                         const float* pool_b, const float* weight_w, const float* weight_b, float* part, float* merge_w, cudaStream_t stream);
/* Branchformer weighted branch average (branchformer_encoder.py:268-276): out = split(w1 * x1 + w2 * x2) [M][D], each product rounded before
 * the add.  (w1, w2) = merge_w[row / Tmax][0..1] (espb_branch_pool_f32), or the constants w1 / w2 when merge_w is NULL (fixed_ave).  x1 / x2
 * rows at stride ldx; D, ldx and out_plane multiples of 4, x1 / x2 / out 16-byte aligned. */
int espb_branch_merge_f32(const float* x1, const float* x2, long long ldx, long long M, int D, int Tmax, const float* merge_w, float w1, float w2,
                          float* out, long long out_plane, cudaStream_t stream);

/* ---- streaming encoder: contextual block processing (espnet2/asr/encoder/contextual_block_conformer_encoder.py:506-572,
 *      legacy/nets/pytorch_backend/conformer/contextual_block_encoder_layer.py:291-308) ---- */
/* chunks [N][nb][block+2][D] from the subsampled frames xs [N][Tt][D]: context token | pos_enc(frames) | context of this block */
int espb_cbe_build_chunks_f32(const float* xs, int N, int Tt, int D, int nb, int block, int hop, const float* pe, int pos0, int ctx0, float scale,
                              const float* prev_addin, float* addin_out, float* chunks, cudaStream_t stream);
/* token 0 of block i := last token of block i-1 (block 0: past_ctx[n][layer] or its own last token); next_ctx[n][layer] := last token of the last block */
int espb_cbe_ctx_propagate_f32(float* x, int N, int nb, int S, int D, const float* past_ctx, float* next_ctx, int layer, int L,
                               cudaStream_t stream);
int espb_zero_rows_f32(float* x, long long row0, long long every, long long count, int D, long long plane, int nplanes, cudaStream_t stream);
int espb_gather_rows_f32(const float* src, int N, long long src_rows, const int* idx, int nout, int D, float* out, cudaStream_t stream);

/* ---- CTC head (espnet2/asr/ctc.py:197-215; greedy collapse asr_inference.py:574-575, s2t_inference_ctc.py:630-632) ---- */
int espb_log_softmax_rows_f32(float* x, long long rows, long long ld, int V, cudaStream_t stream);
int espb_argmax_rows_f32(const float* x, long long rows, long long ld, int V, int* out, cudaStream_t stream);
/* Self-conditioned intermediate CTC: out / out + out_plane [rows][ldo] = tf32 hi / lo of softmax(x[r][0..V-1]) (x row pitch ld), columns
 * V..ldo-1 written as zeros, so the result is the A operand of a 3xTF32 GEMM with K = ldo.  Refused with ESPB_ERR_ARG unless V > 0,
 * ld >= V, ldo >= V with ldo % 32 == 0 and out_plane >= rows * ldo. */
int espb_softmax_rows_split_f32(const float* x, long long rows, long long ld, int V, float* out, long long out_plane, long long ldo,
                                cudaStream_t stream);
int espb_ctc_collapse_i32(const int* argmax, int B, int Tmax, const int* lens, int blank, int* out_ids, int* out_len, cudaStream_t stream);

/* ---- Decoder step (transformer_decoder.py:191-311, decoder_layer.py:73-179, embedding.py:38-95) -------------------------
 * Slots n = U*W (utterance-major). Self-attention cache kc/vc [Lmax][n][D] addressed through anc [n][anc_ld]. */
/* Step-dependent integers (pos / step / out_len) are passed as `value` plus an optional device pointer `step_ptr`: the kernel uses
 * value + *step_ptr when step_ptr != NULL, so one CUDA graph of a decoding step can be replayed for every position. */
int espb_dec_embed_f32(const int* last_tok, const float* emb, const float* pe, int pos, const int* step_ptr, int n, int D, float scale, float* x,
                       cudaStream_t stream);
int espb_dec_self_attn_f32(const float* qkv, float* kc, float* vc, const int* anc, int anc_ld, int n, int D, int H, int pos, const int* step_ptr,
                           int max_pos, float* ctx, long long ctx_plane, cudaStream_t stream);
/* kmem / vmem: [U][H][Tmax][dk] blocks of one decoder layer (projected once per utterance). */
int espb_dec_src_attn_f32(const float* q, const float* kmem, const float* vmem, int U, int Tmax, const int* lens, int W, int D, int H, float* ctx,
                          long long ctx_plane, cudaStream_t stream);

/* ---- Beam search (batch_beam_search.py:253-423, beam_search.py:385-498, e2e_asr_common.py:14-44) -----------------------
 * rows_topk: torch.topk(dim=-1) of x*scale (pre-beam batch_beam_search.py:293-302 and per-row beam candidates). */
int espb_rows_topk_f32(const float* x, long long rows, long long ld, int V, float scale, int k, int* ids, float* vals, cudaStream_t stream);
/* CTCPrefixScoreTH (ctc_prefix_score.py:71-191) + CTCPrefixScorer.select_state (scorers/ctc.py:40-63):
 * r [n][Tmax][4] forward variables per frame (r^n, r^b, r_sum = logaddexp(r^n, r^b), pad), s_prev [n] previous log_psi. */
int espb_ctc_init_state_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int W, float* r, float* s_prev,
                            cudaStream_t stream);
/* CTCPrefixScoreTH.extend_state (ctc_prefix_score.py:251-270): n states [T_old][4] -> [T_new][4] over the extended posteriors logp [T_new][V]
 * of one stream (new frames continue the prefix by blanks only). */
int espb_ctc_extend_state_f32(const float* logp, int T_new, int V, int blank, int n, const float* r_old, int T_old, float* r_new, cudaStream_t stream);
int espb_ctc_score_cands_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int eos, int W, const float* r_prev,
                             const float* s_prev, const int* last_tok, int out_len, const int* step_ptr, const int* cand, int P, float* part,
                             float* psi, int* valid, int token_major, cudaStream_t stream);
int espb_ctc_score_dense_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int eos, int W, const float* r_prev,
                             const float* s_prev, const int* last_tok, int out_len, float* part, cudaStream_t stream);
int espb_ctc_advance_f32(const float* logp, int U, int Tmax, int V, const int* lens, int blank, int eos, int W, const float* r_prev,
                         const int* parent, const int* par_last_tok, const int* new_tok, const int* new_active, int out_len, const int* step_ptr,
                         float* r_new, float* s_new, int token_major, cudaStream_t stream);
/* logp [U][Tmax][V] -> xt [U][V][Tmax]; espb_ctc_score_cands_f32 / espb_ctc_advance_f32 with token_major = 1 read this layout (each
 * candidate's posterior column is then one contiguous, coalesced read instead of a stride-V gather). */
int espb_transpose_tv_f32(const float* x, int U, int Tmax, int V, float* xt, cudaStream_t stream);
/* Weighted sum + beam top-k over (hyps x candidates) per utterance + post_process (eos / maxlen / minlen / end_detect).
 * mode 0 decoder only, 1 joint (pre-beam candidates + eos), 2 CTC only (dense). */
int espb_beam_select(const float* score, const float* sc_dec, const float* sc_ctc, const int* active, float* n_score, float* n_sc_dec,
                     float* n_sc_ctc, int* n_active, int* n_last_tok, int* n_parent, int* bp_parent, int* bp_token, int* ended_count,
                     int* ended_step, int* ended_slot, float* ended_score, float* ended_dec, float* ended_ctc, int ended_cap,
                     float* best_at_step, float* best_all, int* utt_done, int U, int W, int P, int V, int step, const int* step_ptr,
                     const int* maxlen, const int* minlen, int eos, float w_dec, float w_ctc, float penalty, int mode, const int* cand_ids,
                     const float* cand_val, const float* logp_dec, const float* part, const int* valid, int end_detect, int maxlen_cap,
                     cudaStream_t stream);
int espb_anc_update_i32(const int* anc, int* n_anc, int anc_ld, const int* parent, int pos, const int* step_ptr, int n, cudaStream_t stream);
/* ---- LM shallow fusion (espnet2/lm/transformer_lm.py:95-133 as a full scorer; wiring espnet2/bin/asr_inference.py:178-191) ---- */
/* embedding rows of the newest tokens as a split [2][n][E] operand */
int espb_gather_rows_split_f32(const int* tok, const float* emb, int n, int E, float* out, long long plane, cudaStream_t stream);
/* x = relu(x); if pe: x = x * scale + pe[pos (+ *step_ptr)]   (legacy transformer/encoder.py:132-139, embedding.py:85-95) */
int espb_relu_posenc_f32(float* x, int n, int D, const float* pe, int pos, const int* step_ptr, float scale, cudaStream_t stream);
/* out = (wa * a) + (wb * b), products rounded separately: the weighted sum of scorer outputs (batch_beam_search.py:293-300) */
int espb_axpby_f32(const float* a, float wa, const float* b, float wb, float* out, long long n, cudaStream_t stream);
/* per-scorer running scores of the hypotheses chosen by espb_beam_select (merge_scores, beam_search.py:264-293), recorded per step */
int espb_track_scores_f32(const int* parent, const int* tok, const int* bp_parent, const float* logp_a, const float* logp_b, int V, const float* prev_a,
                          const float* prev_b, float* new_a, float* new_b, float* hist_a, float* hist_b, int step, const int* step_ptr, int n,
                          cudaStream_t stream);
/* ---- LSTM LM (espnet2/lm/seq_rnn_lm.py:84-166) as a full scorer.  State ring h, c [2][L][n][Hp] fp32: step pos (+ *step_ptr) reads the
   parent from ring (pos-1)&1 at slot anc[s*anc_ld + pos-1] (zeros at pos 0) and writes ring pos&1 at slot s.  Layer l's GEMM operand is the
   split [2][n][Kp_l] = [input | parent h] with Kp_0 = Ep + Hp, Kp_l = 2*Hp (l >= 1), the L operands back to back in xs; pad columns are
   left untouched (the caller zeroes them once). ---- */
/* embedding row of tok[s] (width E) -> layer 0's input half; parent h of every layer -> that layer's recurrent half */
int espb_rnnlm_gather_f32(const int* tok, const float* emb, int E, int Ep, const int* anc, int anc_ld, int pos, const int* step_ptr,
                          const float* h_ring, int L, int n, int H, int Hp, float* xs, cudaStream_t stream);
/* gates [n][4H] (PyTorch order i, f, g, o) + parent c of layer `layer` -> c' = sig(f) c + sig(i) tanh(g), h' = sig(o) tanh(c') (expf / tanhf)
   into the ring; h' also split into out[s*out_ld + j] (plane out_plane): the next layer's input half or the output projection's operand */
int espb_lstm_cell_f32(const float* gates, const int* anc, int anc_ld, int pos, const int* step_ptr, float* h_ring, float* c_ring, int layer, int L,
                       int n, int H, int Hp, float* out, long long out_plane, int out_ld, cudaStream_t stream);
/* ---- RNN model family (espnet2/asr/encoder/vgg_rnn_encoder.py, rnn_encoder.py, legacy/nets/pytorch_backend/rnn/encoders.py,
 *      asr/decoder/rnn_decoder.py, rnn/attentions.py AttLoc).  The GEMMs (VGG convs as implicit GEMM a_mode 2 over zero-bordered inputs,
 *      input-to-gate products, h W_hh^T, projections, mlp_enc / mlp_dec, decoder gates and output) run on espb_gemm_f32. ---- */
/* VGG2L conv1_1 + ReLU: feats [B][Tf_max][F], utterance b seeing zeros at t >= lens[b] -> split [B][2][F+2][T+2][C] with a zero border
 * and zero rows t >= lens[b] (the input of conv1_2 as implicit GEMM).  w [C][9] ((kt, kf) order), C <= 256. */
int espb_vgg_conv1_relu_f32(const float* feats, int B, int Tf_max, int F, const int* lens, const float* w, const float* bias, int C, float* out,
                            int T, cudaStream_t stream);
/* VGG2L conv output x [B][F][T][C] (plain, ReLU applied), valid at t < lens[b] -> optional 2x2 ceil-mode max-pool over the valid rows
 * (pool = 1: Fo = ceil(F/2), To = ceil(T/2), new length ceil(len/2)) -> flat = 0: split [B][2][Fo+2][To+2][C] zero-bordered (planes
 * out_plane = (Fo+2)(To+2)C apart within an utterance's block); flat = 1: split rows [B*To][C*Fo], column c*Fo + f (the reference's
 * (channel, freq) flattening), planes out_plane apart.  Rows at or past the new length are 0. */
int espb_vgg_pool_f32(const float* x, int B, int F, int T, int C, const int* lens, int pool, int flat, float* out, long long out_plane,
                      cudaStream_t stream);
/* Step s of a 1-layer (B)LSTM over B utterances (packed-sequence semantics): direction d handles frame s (d = 0) or lens[b]-1-s (d = 1).
 * xg [B][T][ndir*4H] input gates with both biases, hg [ndir][B][4H] = h W_hh^T of the previous step (not read at s = 0, where h = c = 0);
 * h' -> h split [2][ndir][B][Hp] (planes h_plane apart), c' -> c [ndir][B][H], h' -> y split [B][T][ldy] columns d*H..; at s >= lens[b]
 * y[b][s] is set to 0 in both directions.  Gate order i, f, g, o; expf / tanhf. */
int espb_lstm_rec_step_f32(const float* xg, const float* hg, const int* lens, int s, int B, int T, int H, int Hp, int ndir, float* h,
                           long long h_plane, float* c, float* y, long long y_plane, int ldy, cudaStream_t stream);
/* Projection epilogue: x [B][T][D] plain -> tanh (act = 1) or identity, rows t >= lens[b] set to 0, into x (write_plain) and / or split
 * into out [B*T][ldo] (out may be NULL). */
int espb_rnn_proj_post_f32(float* x, int B, int T, int D, const int* lens, int act, int write_plain, float* out, long long out_plane, int ldo,
                           cudaStream_t stream);
/* AttLoc step for n = U*W slots (slot s belongs to utterance s / W): previous weights from ring [2][n][Tmax] at (pos-1)&1, slot
 * anc[s*anc_ld + pos-1] (uniform 1/len at pos 0), loc conv (conv_w [chans][2 filts + 1]) + mlp_att (att_wt [chans][A], transposed),
 * e = gvec . tanh(loc + enc_h[u][t] + dec_z[s]) + gvec_b, masked softmax(2 e) over t < lens[u] -> ring[pos&1][s] (0 past len), context
 * sum_t w_t enc[u][t] (enc split [U][Tmax][E], hi + lo) split into out[s*out_ld ..] and, if not NULL, out2[s*out2_ld ..].  enc_h [U][Tmax][A]
 * = mlp_enc(enc).  One block per slot; refused when (Tmax + 2 filts + chans Tmax + Tmax + chans A + 33) floats exceed 227 KiB. */
int espb_att_loc_step_f32(const float* enc_h, const float* enc, long long enc_plane, const int* lens, int W, int Tmax, int A, int E,
                          const float* dec_z, const float* conv_w, int chans, int filts, const float* att_wt, const float* gvec,
                          const float* gvec_b, const int* anc, int anc_ld, int pos, const int* step_ptr, float* ring, int n, float* out,
                          long long out_plane, int out_ld, float* out2, long long out2_plane, int out2_ld, cudaStream_t stream);
/* valid[s*PC + j] = 0 for every slot s < n: drops candidate j (the appended <eos> of espb_ctc_score_cands_f32) for decoders the reference
 * decodes with its non-batch BeamSearch, where <eos> competes only from within the pre-beam (beam_search.py:347-361). */
int espb_drop_cand_i32(int* valid, int n, int PC, int j, cudaStream_t stream);
int espb_step_inc_i32(int* step, cudaStream_t stream);
int espb_count_active_i32(const int* active, int n, int* out, cudaStream_t stream);

/* ---- LM perplexity: full-sequence TransformerLM / SequentialRNNLM forward and ESPnetLanguageModel.nll (espnet2/lm/espnet_model.py:24-70,
   espnet2/bin/lm_calc_perplexity.py) ---- */
/* Causal self-attention of TransformerLM.forward for d_k = 64 (transformer_lm.py:57-72: _target_mask = (ys != 0) & subsequent_mask, through
 * attention.py:153-265): out[b,i,h,:] = softmax_{j <= i, j < len_b, tok[b][j] != 0}( q[b,i,h,:] . k[b,j,h,:] / sqrt(d_k) ) . v[b,j,h,:], a row
 * without a valid key 0.  Layouts and alignment as espb_flash_attn_f32 (no bd); tok [B][T] int32.  Each 128-query block reads only the
 * key tiles up to its last row. */
int espb_causal_flash_attn_f32(const float* q, long long q_off, long long q_plane, long long ldq, const float* k, long long k_off,
                               long long k_plane, long long ldk, const float* vt, long long vt_plane, int Tp, const int* tok, const int* lens, int B,
                               int H, int T, int dk, float* out, long long out_plane, long long ldo, cudaStream_t stream);
/* The same mask for the materialised path (d_k != 64): probs = softmax(scores / sqrt_dk) over the keys j <= i, j < lens[b], tok[b][j] != 0,
 * 0 elsewhere and on rows without a valid key; scores [B][H][T][Tp] -> probs hi/lo planes [B][H][T][Tp]. */
int espb_causal_softmax_f32(const float* scores, int B, int H, int T, int Tp, const int* lens, const int* tok, float sqrt_dk, float* probs,
                            long long probs_plane, cudaStream_t stream);
/* F.cross_entropy(x, tgt, reduction="none") of espnet_model.py:57 in fp32: out[r] = logsumexp(x[r][0..V-1]) - x[r][tgt[r]] (row pitch ld),
 * each row read once with a running max; out[r] = 0 where tgt[r] < 0 (the positions nll zeroes), NaN where tgt[r] >= V. */
int espb_nll_rows_f32(const float* x, long long rows, long long ld, int V, const int* tgt, float* out, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* ESPNET_B200_H */
