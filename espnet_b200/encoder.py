"""ConformerEncoder with the reference's constructor / state_dict surface, executed by the espnet_b200
CUDA kernels (wgmma 3xTF32 GEMMs + warp-primitive glue).

Reference: espnet2/asr/encoder/conformer_encoder.py:89-429 and the legacy modules it composes
(Conv2dSubsampling, RelPositionalEncoding, EncoderLayer, RelPositionMultiHeadedAttention,
PositionwiseFeedForward, ConvolutionModule, LayerNorm).  Supported configuration = the one
BASELINE.json names, with input_layer "conv2d", "conv2d2", "conv2d6" or "conv2d8"; rel_pos_type "latest" (rel_pos / rel_selfattn),
macaron_style, use_cnn_module, swish, normalize_before, intermediate CTC with or without self-conditioning
(interctc_layer_idx / interctc_use_conditioning; no ctc_trim).  The subsampling, FFN, rel-pos self-attention, convolution module and
intermediate-CTC step are the shared ones of layers.py.  The torch.nn layers
are parameter containers only (so that reference checkpoints load by name); forward never calls them.
"""
import math
from typing import List, Optional, Union

import torch

from .layers import LN_EPS, SUBSAMPLING, EncoderBase, _ConvModule, _FFN, _PosBias
# call / ptr / gemm / new_split stay importable here although the shared code in layers.py launches: the kernel emulation of the
# tests replaces these names in every encoder module
from .lib import call, ptr  # noqa: F401
from .ops import ACT_SWISH, gemm, layernorm, linear, new_split  # noqa: F401


class _EncoderLayer(torch.nn.Module):
    def __init__(self, d, heads, units, kernel):
        super().__init__()
        self.self_attn = _PosBias(heads, d)
        self.feed_forward = _FFN(d, units)
        self.feed_forward_macaron = _FFN(d, units)
        self.conv_module = _ConvModule(d, kernel)
        self.norm_ff = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_mha = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_ff_macaron = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_conv = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_final = torch.nn.LayerNorm(d, eps=LN_EPS)


class ConformerEncoder(EncoderBase):
    """Drop-in for espnet2.asr.encoder.conformer_encoder.ConformerEncoder (inference, CUDA only)."""

    def __init__(self, input_size: int, output_size: int = 256, attention_heads: int = 4, linear_units: int = 2048,
                 num_blocks: int = 6, dropout_rate: float = 0.1, positional_dropout_rate: float = 0.1,
                 attention_dropout_rate: float = 0.0, input_layer: Optional[str] = "conv2d", normalize_before: bool = True,
                 concat_after: bool = False, positionwise_layer_type: str = "linear", positionwise_conv_kernel_size: int = 3,
                 macaron_style: bool = False, rel_pos_type: str = "legacy", pos_enc_layer_type: str = "rel_pos",
                 selfattention_layer_type: str = "rel_selfattn", activation_type: str = "swish", use_cnn_module: bool = True,
                 zero_triu: bool = False, cnn_module_kernel: int = 31, padding_idx: int = -1, interctc_layer_idx: List[int] = [],
                 interctc_use_conditioning: bool = False, ctc_trim: bool = False,
                 stochastic_depth_rate: Union[float, List[float]] = 0.0, layer_drop_rate: float = 0.0,
                 max_pos_emb_len: int = 5000, qk_norm: bool = False, use_flash_attn: bool = True):
        unsupported = []
        if input_layer not in SUBSAMPLING: unsupported.append(f"input_layer={input_layer}")
        if rel_pos_type != "latest" or pos_enc_layer_type != "rel_pos" or selfattention_layer_type != "rel_selfattn":
            unsupported.append("rel_pos_type/pos_enc_layer_type/selfattention_layer_type other than latest/rel_pos/rel_selfattn")
        if not (normalize_before and macaron_style and use_cnn_module) or concat_after: unsupported.append("non pre-LN macaron+cnn block")
        if positionwise_layer_type != "linear" or activation_type != "swish": unsupported.append("positionwise/activation type")
        if zero_triu or qk_norm or ctc_trim: unsupported.append("zero_triu/qk_norm/ctc_trim")
        if cnn_module_kernel < 1 or cnn_module_kernel % 2 == 0 or cnn_module_kernel > 127:
            unsupported.append(f"cnn_module_kernel={cnn_module_kernel} (odd, <= 127)")
        if unsupported:
            raise NotImplementedError("espnet_b200 ConformerEncoder supports the BASELINE configuration only; got " + ", ".join(unsupported))
        assert output_size % attention_heads == 0
        if output_size % 32:
            raise NotImplementedError("espnet_b200 ConformerEncoder: output_size must be a multiple of 32")
        super().__init__(input_size, output_size,
                         (_EncoderLayer(output_size, attention_heads, linear_units, cnn_module_kernel) for _ in range(num_blocks)), input_layer)
        self.heads, self.num_blocks, self.kernel = attention_heads, num_blocks, cnn_module_kernel
        self._init_interctc(interctc_layer_idx, interctc_use_conditioning, num_blocks)

    def _pack(self):
        pk = self._pack_io()
        layers = []
        for lyr in self.encoders:
            d = {nm: self._pack_ln(getattr(lyr, nm)) for nm in ("norm_ff_macaron", "norm_mha", "norm_conv", "norm_ff", "norm_final")}
            d["feed_forward_macaron"], d["feed_forward"] = self._pack_ffn(lyr.feed_forward_macaron), self._pack_ffn(lyr.feed_forward)
            d.update(self._pack_mha(lyr.self_attn), **self._pack_conv(lyr.conv_module))
            layers.append(d)
        pk["layers"] = layers
        pk["pos_w_all"] = self._pack_pos(lyr.self_attn for lyr in self.encoders)
        self._packed = pk
        return pk

    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None, ctc=None):
        """xs_pad (B, T_f, idim) float32 CUDA (normalised log-mel), ilens (B,) -> (B, T, D), olens, None; with interctc_layer_idx
        ((B, T, D), [(layer, after_norm of that block's output), ...]), olens, None.  ctc: the CTC head, needed with
        interctc_use_conditioning.

        Ragged batches follow per-utterance (batch-1) semantics of the reference: every utterance sees only
        its own frames (own conv boundaries, own attention keys); rows t >= olens[b] of the output are padding."""
        self._check_interctc(ctc)
        pk = self._packed or self._pack()
        xs_pad, T, olens, lens32 = self._lengths(xs_pad, ilens)   # check_short_utt: conformer_encoder.py:363-371
        B, D = xs_pad.shape[0], self._output_size
        M = B * T
        x = self._buf("x", (M, D))
        self._subsample(xs_pad, x, math.sqrt(D))
        if self.trace is not None:
            self.trace.append(x.view(B, T, D).clone())
        p_all = self._pos(T)
        xn, qkv, ctx = self._buf("xn", (2, M, D)), self._buf("qkv", (2, M, 3 * D)), self._buf("ctx", (2, M, D))
        inter = []
        for li, w in enumerate(pk["layers"]):
            # macaron FFN: x += 0.5 * w2(swish(w1(LN(x))))   (encoder_layer.py:115-123)
            self._ffn(x, xn, w["norm_ff_macaron"], w["feed_forward_macaron"], ACT_SWISH, 0.5)
            # rel-pos MHSA (encoder_layer.py:126-149)
            layernorm(x, *w["norm_mha"], LN_EPS, out_split=xn)
            linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
            self._relpos_attn(qkv, w, li, p_all, ctx, B, T, lens32)
            linear(ctx, w["out_w"], x, bias=w["out_b"], residual=x)
            # convolution module (encoder_layer.py:152-158)
            self._conv_module(x, xn, w["norm_conv"], w, B, T, lens32)
            # FFN + final norm (encoder_layer.py:161-171)
            self._ffn(x, xn, w["norm_ff"], w["feed_forward"], ACT_SWISH, 0.5)
            layernorm(x, *w["norm_final"], LN_EPS, out_plain=x)
            if self.trace is not None:
                self.trace.append(x.view(B, T, D).clone())
            if li + 1 in self.interctc_layer_idx:
                inter.append((li + 1, self._interctc(x, B, T, ctc)))
        out, _ = self._output(x, B, T)
        return ((out, inter) if inter else out), olens, None
