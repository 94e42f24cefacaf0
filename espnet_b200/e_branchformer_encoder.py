"""EBranchformerEncoder with the reference's constructor / state_dict surface, executed by the espnet_b200 CUDA kernels.

Reference: espnet2/asr/encoder/e_branchformer_encoder.py:55-563 (EBranchformerEncoderLayer, EBranchformerEncoder) and
espnet2/asr/layers/cgmlp.py:15-124 (ConvolutionalSpatialGatingUnit, ConvolutionalGatingMLP).  The subsampling, the FFNs and the attention
branch are the shared ones of layers.py -- the Conformer's rel-pos "latest" self-attention (band GEMM over a cached P_all, then the fused
wgmma attention at d_k = 64); the cgMLP branch, shared with the Branchformer in layers.py, is
channel_proj1 with GELU in the GEMM epilogue, the CSGU kernel (LayerNorm + depthwise conv + gating, csrc/encoder_ops.cu) and
channel_proj2; the merge module is one depthwise-conv kernel over the concatenated branches followed by merge_proj.

Both branches write plain fp32 into one [M, 2D] buffer: the attention output (linear_out) into columns [0, D), channel_proj2 into
columns [D, 2D) -- the torch.cat of the reference.  The torch.nn layers are parameter containers only (reference checkpoints load by
name); forward never calls them.
"""
import math
from typing import List, Optional, Tuple

import torch

from .layers import LN_EPS, SUBSAMPLING, EncoderBase, _CgMLP, _FFN, _PosBias
# new_split stays importable here although _pos in layers.py allocates: the kernel emulation of the tests replaces it in this module
from .lib import call, ptr
from .ops import ACT_GELU, ACT_RELU, ACT_SWISH, _count, gemm, layernorm, linear, new_split, split_from  # noqa: F401

_FFN_ACTS = {"swish": ACT_SWISH, "relu": ACT_RELU}   # get_activation (nets_utils.py:571-584) choices this path computes


class _Layer(torch.nn.Module):
    def __init__(self, d, heads, cgmlp_units, cgmlp_kernel, ffn_units, use_ffn, macaron, merge_kernel):
        super().__init__()
        self.attn = _PosBias(heads, d)
        self.cgmlp = _CgMLP(d, cgmlp_units, cgmlp_kernel)
        self.feed_forward = _FFN(d, ffn_units) if use_ffn else None
        self.feed_forward_macaron = _FFN(d, ffn_units) if use_ffn and macaron else None
        if use_ffn:
            self.norm_ff = torch.nn.LayerNorm(d, eps=LN_EPS)
        if use_ffn and macaron:
            self.norm_ff_macaron = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_mha = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_mlp = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_final = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.depthwise_conv_fusion = torch.nn.Conv1d(2 * d, 2 * d, merge_kernel, 1, (merge_kernel - 1) // 2, groups=2 * d)
        self.merge_proj = torch.nn.Linear(2 * d, d)


class EBranchformerEncoder(EncoderBase):
    """Drop-in for espnet2.asr.encoder.e_branchformer_encoder.EBranchformerEncoder (inference, CUDA only)."""

    def __init__(self, input_size: int, output_size: int = 256, attention_heads: int = 4, attention_layer_type: str = "rel_selfattn",
                 pos_enc_layer_type: str = "rel_pos", rel_pos_type: str = "latest", cgmlp_linear_units: int = 2048, cgmlp_conv_kernel: int = 31,
                 use_linear_after_conv: bool = False, gate_activation: str = "identity", num_blocks: int = 12, dropout_rate: float = 0.1,
                 positional_dropout_rate: float = 0.1, attention_dropout_rate: float = 0.0, input_layer: Optional[str] = "conv2d",
                 zero_triu: bool = False, padding_idx: int = -1, layer_drop_rate: float = 0.0, max_pos_emb_len: int = 5000,
                 use_ffn: bool = False, macaron_ffn: bool = False, ffn_activation_type: str = "swish", linear_units: int = 2048,
                 positionwise_layer_type: str = "linear", merge_conv_kernel: int = 3, interctc_layer_idx=None,
                 interctc_use_conditioning: bool = False, qk_norm: bool = False, use_flash_attn: bool = True,
                 gradient_checkpoint_layers: List[int] = []):
        unsupported = []
        if input_layer not in SUBSAMPLING: unsupported.append(f"input_layer={input_layer}")
        if rel_pos_type != "latest" or pos_enc_layer_type != "rel_pos" or attention_layer_type != "rel_selfattn":
            unsupported.append("rel_pos_type/pos_enc_layer_type/attention_layer_type other than latest/rel_pos/rel_selfattn")
        if use_linear_after_conv or gate_activation != "identity": unsupported.append("use_linear_after_conv / non-identity gate_activation")
        if use_ffn and (positionwise_layer_type != "linear" or ffn_activation_type not in _FFN_ACTS):
            unsupported.append(f"positionwise_layer_type={positionwise_layer_type} / ffn_activation_type={ffn_activation_type}")
        for name, k in (("cgmlp_conv_kernel", cgmlp_conv_kernel), ("merge_conv_kernel", merge_conv_kernel)):
            if k < 1 or k % 2 == 0 or k > 127: unsupported.append(f"{name}={k} (odd, <= 127)")
        if cgmlp_linear_units % 2 or cgmlp_linear_units // 2 > 2048: unsupported.append(f"cgmlp_linear_units={cgmlp_linear_units} (even, <= 4096)")
        if zero_triu or qk_norm or interctc_layer_idx: unsupported.append("zero_triu/qk_norm/interctc")
        if unsupported:
            raise NotImplementedError("espnet_b200 EBranchformerEncoder does not support: " + ", ".join(unsupported))
        assert output_size % attention_heads == 0
        if output_size % 32:
            raise NotImplementedError("espnet_b200 EBranchformerEncoder: output_size must be a multiple of 32")
        super().__init__(input_size, output_size, (
            _Layer(output_size, attention_heads, cgmlp_linear_units, cgmlp_conv_kernel, linear_units, use_ffn, macaron_ffn, merge_conv_kernel)
            for _ in range(num_blocks)), input_layer)
        self.heads, self.num_blocks = attention_heads, num_blocks
        self.cgmlp_units, self.cgmlp_kernel, self.merge_kernel = cgmlp_linear_units, cgmlp_conv_kernel, merge_conv_kernel
        self.use_ffn, self.macaron = use_ffn, use_ffn and macaron_ffn
        self.ffn_act = _FFN_ACTS.get(ffn_activation_type, ACT_SWISH)
        self.ff_scale = 0.5 if self.macaron else 1.0

    def _pack(self):
        pk = self._pack_io()
        f32, ln, D = self._f32, self._pack_ln, self._output_size
        layers = []
        for lyr in self.encoders:
            d = dict(norm_mha=ln(lyr.norm_mha), norm_mlp=ln(lyr.norm_mlp), norm_final=ln(lyr.norm_final))
            if self.use_ffn:
                d["norm_ff"], d["ffn"] = ln(lyr.norm_ff), self._pack_ffn(lyr.feed_forward)
            if self.macaron:
                d["norm_ff_macaron"], d["ffn_macaron"] = ln(lyr.norm_ff_macaron), self._pack_ffn(lyr.feed_forward_macaron)
            d.update(self._pack_mha(lyr.attn))
            d.update(self._pack_cgmlp(lyr.cgmlp))
            d["mg_w"], d["mg_b"] = f32(lyr.depthwise_conv_fusion.weight).view(2 * D, -1), f32(lyr.depthwise_conv_fusion.bias)
            d["mp_w"], d["mp_b"] = split_from(f32(lyr.merge_proj.weight)), f32(lyr.merge_proj.bias)
            layers.append(d)
        pk["layers"] = layers
        pk["pos_w_all"] = self._pack_pos(lyr.attn for lyr in self.encoders)
        self._packed = pk
        return pk

    # ---------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """xs_pad (B, T_f, idim) float32 CUDA (normalised log-mel), ilens (B,) -> (B, T, D), olens, None.

        Ragged batches follow per-utterance (batch-1) semantics of the reference: every utterance sees only its own frames (own attention
        keys, own conv boundaries in the CSGU and the merge module); rows t >= olens[b] of the output are 0."""
        pk = self._packed or self._pack()
        xs_pad, T, olens, lens32 = self._lengths(xs_pad, ilens)   # check_short_utt: e_branchformer_encoder.py:482-499
        B, D = xs_pad.shape[0], self._output_size
        M = B * T
        x = self._buf("x", (M, D))
        self._subsample(xs_pad, x, math.sqrt(D))
        if self.trace is not None:
            self.trace.append(x.view(B, T, D).clone())
        p_all = self._pos(T)

        xn, qkv, ctx = self._buf("xn", (2, M, D)), self._buf("qkv", (2, M, 3 * D)), self._buf("ctx", (2, M, D))
        cat = self._buf("cat", (M, 2 * D))        # [x_att | x_cgmlp], plain
        mg = self._buf("mg", (2, M, 2 * D))       # cat + dwconv(cat), split
        for li, w in enumerate(pk["layers"]):
            if self.macaron:
                self._ffn(x, xn, w["norm_ff_macaron"], w["ffn_macaron"], self.ffn_act, self.ff_scale)
            # branch 1: rel-pos MHSA (e_branchformer_encoder.py:141-152, attention.py:416-459) -> cat[:, :D]
            layernorm(x, *w["norm_mha"], LN_EPS, out_split=xn)
            linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
            self._relpos_attn(qkv, w, li, p_all, ctx, B, T, lens32)
            gemm(M, D, D, ctx, M * D, D, w["out_w"], D * D, D, cat, 2 * D, bias=w["out_b"])
            # branch 2: cgMLP (e_branchformer_encoder.py:154-163, cgmlp.py:110-124) -> cat[:, D:]
            self._cgmlp(x, xn, w, B, T, lens32, cat, 2 * D, c_off=D)
            # merge: x += merge_proj(cat + dwconv(cat))  (e_branchformer_encoder.py:165-170)
            call("espb_merge_dwconv_f32", ptr(cat), B, T, 2 * D, ptr(lens32), ptr(w["mg_w"]), ptr(w["mg_b"]), self.merge_kernel, ptr(mg), M * 2 * D)
            _count()
            linear(mg, w["mp_w"], x, bias=w["mp_b"], residual=x)
            if self.use_ffn:
                self._ffn(x, xn, w["norm_ff"], w["ffn"], self.ffn_act, self.ff_scale)
            layernorm(x, *w["norm_final"], LN_EPS, out_plain=x)
            if self.trace is not None:
                self.trace.append(x.view(B, T, D).clone())
        out, out_split = self._output(x, B, T)
        call("espb_zero_pad_rows_f32", ptr(out), B, T, D, ptr(lens32), 0, 1)
        call("espb_zero_pad_rows_f32", ptr(out_split), B, T, D, ptr(lens32), M * D, 2)
        _count(2)
        return out, olens, None
