"""ctypes binding of the C-ABI library ``libespnet_b200.so`` (see include/espnet_b200.h).

The library is plain CUDA C++ with ``extern "C"`` entry points taking raw device pointers, sizes
and a ``cudaStream_t``; PyTorch only provides the device buffers and the stream.  There is no CPU
fallback: importing succeeds without the library (so CPU-only tooling can import the package), but
every op raises if the library is missing.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_float, c_int, c_longlong, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libespnet_b200.so")

_lib = None


class GemmDesc(Structure):
    """Mirror of EspbGemmDesc (espnet_b200/csrc/gemm.h)."""

    _fields_ = [
        ("M", c_int), ("N", c_int), ("K", c_int), ("nbx", c_int), ("nby", c_int), ("a_mode", c_int), ("kob", c_int),
        ("A", c_void_p), ("a_plane", c_longlong), ("lda", c_longlong), ("sa_x", c_longlong), ("sa_y", c_longlong),
        ("B", c_void_p), ("b_plane", c_longlong), ("ldb", c_longlong), ("sb_x", c_longlong), ("sb_y", c_longlong),
        ("C", c_void_p), ("c_plane", c_longlong), ("ldc", c_longlong), ("sc_x", c_longlong), ("sc_y", c_longlong),
        ("split_out", c_int), ("bias", c_void_p), ("sbias_x", c_longlong),
        ("R", c_void_p), ("ldr", c_longlong), ("sr_x", c_longlong), ("sr_y", c_longlong),
        ("alpha", c_float), ("act", c_int), ("cv_t1h", c_int), ("cv_f1h", c_int), ("cv_cin", c_int), ("band_t", c_int),
    ]


P, I, L, F = c_void_p, c_int, c_longlong, c_float

# name -> argtypes (all return int status); mirrors include/espnet_b200.h
_SIGS = {
    "espb_gemm_f32": [POINTER(GemmDesc), I, P],
    "espb_stft_logmel_f32": [P, P, I, I, I, P, P, P, P, P, P, P, I, I, P, I, P, P],
    "espb_utt_mvn_from_partial_f32": [P, P, I, I, I, I, P, P],
    "espb_utt_mvn_f32": [P, P, I, I, I, P, P],
    "espb_global_mvn_f32": [P, P, I, I, I, P, P, I, I, P],
    "espb_layernorm_f32": [P, L, I, P, P, F, P, P, L, P],
    "espb_split_tf32_f32": [P, L, P, L, P],
    "espb_conv1_relu_f32": [P, I, I, I, P, P, I, P, I, I, I, I, P],
    "espb_conv1_relu_phase_f32": [P, I, I, I, P, P, I, P, I, I, I, I, I, P],
    "espb_phase_split_f32": [P, L, I, I, I, I, I, I, I, P, P],
    "espb_qu_qv_f32": [P, L, L, I, P, P, P, P, L, P],
    "espb_v_transpose_f32": [P, L, I, I, I, I, P, P, L, I, P],
    "espb_relpos_softmax_f32": [P, P, I, I, I, I, I, P, F, P, L, P],
    "espb_masked_softmax_f32": [P, I, I, I, I, P, F, P, L, P],
    "espb_flash_attn_f32": [P, L, L, L, P, L, L, L, P, L, I, P, I, P, I, I, I, I, P, L, L, P],
    "espb_glu_dwconv_bn_swish_f32": [P, I, I, I, P, P, P, I, P, P, P, L, P],
    "espb_zero_pad_rows_f32": [P, I, I, I, P, L, I, P],
    "espb_csgu_f32": [P, I, I, I, P, P, P, F, P, P, I, P, P, L, P],
    "espb_merge_dwconv_f32": [P, I, I, I, P, P, P, I, P, L, P],
    "espb_branch_pool_f32": [P, P, L, I, I, I, P, P, P, P, P, P, P, P],
    "espb_branch_merge_f32": [P, P, L, L, I, I, P, F, F, P, L, P],
    "espb_cbe_build_chunks_f32": [P, I, I, I, I, I, I, P, I, I, F, P, P, P, P],
    "espb_cbe_ctx_propagate_f32": [P, I, I, I, I, P, P, I, I, P],
    "espb_zero_rows_f32": [P, L, L, L, I, L, I, P],
    "espb_gather_rows_f32": [P, I, L, P, I, I, P, P],
    "espb_log_softmax_rows_f32": [P, L, L, I, P],
    "espb_argmax_rows_f32": [P, L, L, I, P, P],
    "espb_softmax_rows_split_f32": [P, L, L, I, P, L, L, P],
    "espb_ctc_collapse_i32": [P, I, I, P, I, P, P, P],
    "espb_dec_embed_f32": [P, P, P, I, P, I, I, F, P, P],
    "espb_dec_self_attn_f32": [P, P, P, P, I, I, I, I, I, P, I, P, L, P],
    "espb_dec_src_attn_f32": [P, P, P, I, I, P, I, I, I, P, L, P],
    "espb_rows_topk_f32": [P, L, L, I, F, I, P, P, P],
    "espb_ctc_init_state_f32": [P, I, I, I, P, I, I, P, P, P],
    "espb_ctc_extend_state_f32": [P, I, I, I, I, P, I, P, P],
    "espb_ctc_score_cands_f32": [P, I, I, I, P, I, I, I, P, P, P, I, P, P, I, P, P, P, I, P],
    "espb_ctc_score_dense_f32": [P, I, I, I, P, I, I, I, P, P, P, I, P, P],
    "espb_beam_select": [P] * 18 + [I] + [P, P, P] + [I, I, I, I, I, P, P, P, I, F, F, F, I, P, P, P, P, P, I, I, P],
    "espb_anc_update_i32": [P, P, I, P, I, P, I, P],
    "espb_step_inc_i32": [P, P],
    "espb_gather_rows_split_f32": [P, P, I, I, P, L, P],
    "espb_relu_posenc_f32": [P, I, I, P, I, P, F, P],
    "espb_axpby_f32": [P, F, P, F, P, L, P],
    "espb_track_scores_f32": [P, P, P, P, P, I, P, P, P, P, P, P, I, P, I, P],
    "espb_ctc_advance_f32": [P, I, I, I, P, I, I, I, P, P, P, P, P, I, P, P, P, I, P],
    "espb_transpose_tv_f32": [P, I, I, I, P, P],
    "espb_count_active_i32": [P, I, P, P],
    "espb_rnnlm_gather_f32": [P, P, I, I, P, I, I, P, P, I, I, I, I, P, P],
    "espb_lstm_cell_f32": [P, P, I, I, P, P, P, I, I, I, I, I, P, L, I, P],
    "espb_vgg_conv1_relu_f32": [P, I, I, I, P, P, P, I, P, I, P],
    "espb_vgg_pool_f32": [P, I, I, I, I, P, I, I, P, L, P],
    "espb_lstm_rec_step_f32": [P, P, P, I, I, I, I, I, I, P, L, P, P, L, I, P],
    "espb_rnn_proj_post_f32": [P, I, I, I, P, I, I, P, L, I, P],
    "espb_drop_cand_i32": [P, I, I, I, P],
    "espb_att_loc_step_f32": [P, P, L, P, I, I, I, I, P, P, I, I, P, P, P, P, I, I, P, P, I, P, L, I, P, L, I, P],
    "espb_causal_flash_attn_f32": [P, L, L, L, P, L, L, L, P, L, I, P, P, I, I, I, I, P, L, L, P],
    "espb_causal_softmax_f32": [P, I, I, I, I, P, P, F, P, L, P],
    "espb_nll_rows_f32": [P, L, L, I, P, P, P],
}

ABI_VERSION = 7   # espb_abi_version() of the library this binding matches (include/espnet_b200.h)
EXPORTED_SYMBOLS = sorted(list(_SIGS) + ["espb_last_error", "espb_abi_version", "espb_device_sm", "espb_frontend_blocks"])


class LibraryMissing(RuntimeError):
    pass


def load():
    """Load (once) and return the ctypes handle; raises LibraryMissing if the .so is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C espnet_b200/csrc`). There is no CPU fallback for the espnet_b200 ops.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, args in _SIGS.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = c_int
    lib.espb_last_error.restype = ctypes.c_char_p
    lib.espb_last_error.argtypes = []
    lib.espb_abi_version.restype = c_int
    if lib.espb_abi_version() != ABI_VERSION:
        raise LibraryMissing(f"{LIB_PATH} has ABI version {lib.espb_abi_version()}, this package binds version {ABI_VERSION}: rebuild it "
                             "(`make -C espnet_b200/csrc`)")
    lib.espb_frontend_blocks.argtypes = [c_int]
    lib.espb_frontend_blocks.restype = c_int
    lib.espb_device_sm.argtypes = [POINTER(c_int), POINTER(c_int)]
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().espb_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"espnet_b200 {what} failed (code {rc}): {msg}")


def ptr(t):
    """Device pointer of a tensor (or None)."""
    if t is None:
        return None
    assert t.is_cuda, "espnet_b200 ops need CUDA tensors (no CPU fallback)"
    return c_void_p(t.data_ptr())


def stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


profile = None  # set to a list to record (name, tag, start_event, end_event) for every launch (bench --breakdown)
profile_tag = [""]


def call(name, *args):
    lib = load()
    if profile is None:
        check(getattr(lib, name)(*args, stream()), name)
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    check(getattr(lib, name)(*args, stream()), name)
    e1.record()
    profile.append((name, profile_tag[0], e0, e1))
    profile_tag[0] = ""
