"""Python-side launch helpers over the C-ABI (espnet_b200/lib.py).  No compute happens here.

Split tensors: a tensor that feeds a tensor-core GEMM is stored as two fp32 planes ``t[0]`` (tf32
"hi") and ``t[1]`` ("lo"), shape ``[2, ...]`` contiguous; see espnet_b200/csrc/gemm.h.
"""
import os

import torch

from . import lib
from .lib import GemmDesc, call, ptr

ACT_NONE, ACT_RELU, ACT_SWISH, ACT_GELU = 0, 1, 2, 3

# GEMM kernel: "tc" = wgmma 3xTF32, "tc2" = wgmma 3xTF32 with chunked fp32 promotion, "simt" = FFMA (bring-up / A-B checks);
# shapes TMA cannot address always use SIMT.
_GEMM_MODE = os.environ.get("ESPNET_B200_GEMM", "tc2")
launch_counter = [0]
gemm_profile = None  # set to a list to record (algorithmic flops, start event, end event) per tensor-core GEMM launch


def set_gemm_mode(mode):
    global _GEMM_MODE
    assert mode in ("tc", "tc2", "simt")
    _GEMM_MODE = mode


def gemm_mode():
    return _GEMM_MODE


def _count(n=1):
    launch_counter[0] += n


def new_split(*shape, device="cuda"):
    return torch.empty((2,) + tuple(shape), dtype=torch.float32, device=device)


def split_from(x):
    """fp32 tensor -> split tensor [2, *x.shape] on device."""
    x = x.contiguous()
    out = new_split(*x.shape, device=x.device)
    call("espb_split_tf32_f32", ptr(x), x.numel(), ptr(out), x.numel())
    _count()
    return out


def gemm(M, N, K, A, a_plane, lda, B, b_plane, ldb, C, ldc, *, c_plane=0, split_out=False, bias=None, R=None, ldr=0,
         alpha=1.0, act=ACT_NONE, nbx=1, nby=1, sa=(0, 0), sb=(0, 0), sc=(0, 0), sr=(0, 0), kob=0, a_mode=0, conv=(0, 0, 0),
         a_off=0, b_off=0, c_off=0, r_off=0, sbias_x=0, bias_off=0, band_t=0, force=None):
    """Raw strided GEMM launch; A/B/C/R are tensors (base pointers), *_off element offsets."""
    d = GemmDesc()
    d.M, d.N, d.K, d.nbx, d.nby, d.a_mode, d.kob = M, N, K, nbx, nby, a_mode, kob
    d.A = A.data_ptr() + 4 * a_off
    d.a_plane, d.lda, d.sa_x, d.sa_y = a_plane, lda, sa[0], sa[1]
    d.B = B.data_ptr() + 4 * b_off
    d.b_plane, d.ldb, d.sb_x, d.sb_y = b_plane, ldb, sb[0], sb[1]
    d.C = C.data_ptr() + 4 * c_off
    d.c_plane, d.ldc, d.sc_x, d.sc_y = c_plane, ldc, sc[0], sc[1]
    d.split_out = 1 if split_out else 0
    d.bias = (bias.data_ptr() + 4 * bias_off) if bias is not None else None
    d.sbias_x = sbias_x
    d.R = (R.data_ptr() + 4 * r_off) if R is not None else None
    d.ldr, d.sr_x, d.sr_y = ldr, sr[0], sr[1]
    d.alpha, d.act = float(alpha), act
    d.cv_t1h, d.cv_f1h, d.cv_cin = conv
    d.band_t = band_t
    mode = force or _GEMM_MODE
    use_tc = {"tc": 1, "tc2": 2}.get(mode, 0)
    if use_tc:
        # TMA needs 16-byte aligned bases and strides
        al = [lda, ldb, a_plane, b_plane, sa[0], sa[1], sb[0], sb[1], a_off, b_off]
        if any(v % 4 for v in al):
            use_tc = 0
        if a_mode and conv[2] % 32:
            use_tc = 0
        if a_mode == 0 and kob > 0 and K % (kob * 32):
            use_tc = 0
    if lib.profile is not None:
        lib.profile_tag[0] = f"{'tc' + str(use_tc) if use_tc else 'simt'} M{M} N{N} K{K} x{nbx * nby}" + (" conv" if a_mode else "")
    prof = gemm_profile if use_tc else None
    if prof is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    call("espb_gemm_f32", d, use_tc)
    if prof is not None:
        e1.record()
        n_alg = band_t if band_t > 0 else N     # rel-pos band product: every row needs band_t of the N columns
        prof.append((2.0 * M * n_alg * K * nbx * nby, e0, e1))
    _count()
    return bool(use_tc)


def linear(x_split, w_split, out, *, bias=None, act=ACT_NONE, residual=None, alpha=1.0, split_out=False, force=None):
    """out[M,N] = epilogue(x[M,K] @ w[N,K]^T).  x_split [2,M,K], w_split [2,N,K]; out [M,N] or [2,M,N]."""
    M, K = x_split.shape[1], x_split.shape[2]
    N = w_split.shape[1]
    assert w_split.shape[2] == K
    return gemm(M, N, K, x_split, M * K, K, w_split, N * K, K, out, N, c_plane=M * N, split_out=split_out, bias=bias,
                R=residual, ldr=N, alpha=alpha, act=act, force=force)


# Fused wgmma self-attention (csrc/attention.cu) for d_k = 64; ESPB_ATTN=materialized keeps the round-1 GEMM + softmax + GEMM sequence
# (A/B measurements and the validator of the fused kernel).
_ATTN_MODE = os.environ.get("ESPB_ATTN", "fused")


def set_attn_mode(mode):
    global _ATTN_MODE
    assert mode in ("fused", "materialized")
    _ATTN_MODE = mode


def attn_mode():
    return _ATTN_MODE


def use_flash_attn(dk):
    return _ATTN_MODE == "fused" and dk == 64 and _GEMM_MODE != "simt"


def flash_attn(q_split, q_off, ldq, k_split, k_off, ldk, vt, Tp, bd, Rp, lens32, B, H, T, dk, out_split):
    """out_split [2][B*T][H*dk] = softmax((q k^T + rel_shift(bd)) / sqrt(dk)) v per (utterance, head); bd None: plain attention."""
    call("espb_flash_attn_f32", ptr(q_split), q_off, q_split[0].numel(), ldq, ptr(k_split), k_off, k_split[0].numel(), ldk, ptr(vt),
         vt[0].numel(), Tp, ptr(bd), Rp, ptr(lens32), B, H, T, dk, ptr(out_split), out_split[0].numel(), H * dk)
    _count()


def layernorm(x, gamma, beta, eps, out_plain=None, out_split=None):
    rows, D = x.numel() // x.shape[-1], x.shape[-1]
    plane = out_split[0].numel() if out_split is not None else 0
    call("espb_layernorm_f32", ptr(x), rows, D, ptr(gamma), ptr(beta), eps, ptr(out_plain), ptr(out_split), plane)
    _count()


def log_softmax_rows_(x2d):
    call("espb_log_softmax_rows_f32", ptr(x2d), x2d.shape[0], x2d.stride(0), x2d.shape[1])
    _count()


def softmax_rows_split(x2d, out_split):
    """out_split [2][rows][ldo] = tf32 hi / lo of the row softmax of x2d [rows][V]; columns V..ldo-1 zero (ldo % 32 == 0)."""
    call("espb_softmax_rows_split_f32", ptr(x2d), x2d.shape[0], x2d.stride(0), x2d.shape[1], ptr(out_split), out_split[0].numel(),
         out_split.shape[2])
    _count()


def argmax_rows(x2d, out):
    call("espb_argmax_rows_f32", ptr(x2d), x2d.shape[0], x2d.stride(0), x2d.shape[1], ptr(out))
    _count()


def rows_topk(x2d, scale, k, ids, vals):
    call("espb_rows_topk_f32", ptr(x2d), x2d.shape[0], x2d.stride(0), x2d.shape[1], float(scale), k, ptr(ids), ptr(vals))
    _count()
