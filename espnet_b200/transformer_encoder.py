"""TransformerEncoder (absolute positions, conv2d / conv2d2 / conv2d6 / conv2d8 input layer, pre-LN, ReLU feed-forward) with the reference's constructor /
state_dict surface -- the encoder of the next scope row (SURVEY.md 8f-1, BASELINE configs[4]), with intermediate CTC and self-conditioning (interctc_layer_idx / interctc_use_conditioning).  It composes the kernels of the
Conformer path (conv1 / implicit-GEMM conv2 / wgmma 3xTF32 GEMMs / LayerNorm) plus a plain masked softmax; the subsampling, FFN and
self-attention are the shared ones of layers.py.

Reference: espnet2/asr/encoder/transformer_encoder.py:43-299, legacy/nets/pytorch_backend/transformer/encoder_layer.py:65-126,
attention.py:77-151,262-265 (default branch), embedding.py:38-95 (PositionalEncoding), subsampling.py:386-862.
Parity: tests/test_gpu_zz_next.py (reference fixture layer by layer, ragged batch, whole Speech2Text) and tests/test_host_logic_emulated.py; self-attention
is the fused wgmma kernel without the rel-pos term (csrc/attention.cu) at d_k = 64.
"""
import math
from typing import List, Optional

import torch

from . import ops
from .layers import LN_EPS, SUBSAMPLING, EncoderBase, _FFN, _MHA, abs_pos_table
# call / ptr / gemm stay importable here although the shared code in layers.py launches: the kernel emulation of the tests replaces
# these names in every encoder module
from .lib import call, ptr  # noqa: F401
from .ops import ACT_RELU, gemm, layernorm, linear  # noqa: F401


class _Layer(torch.nn.Module):
    def __init__(self, d, units):
        super().__init__()
        self.self_attn = _MHA(d)
        self.feed_forward = _FFN(d, units)
        self.norm1 = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm2 = torch.nn.LayerNorm(d, eps=LN_EPS)


class TransformerEncoder(EncoderBase):
    """Drop-in for espnet2.asr.encoder.transformer_encoder.TransformerEncoder (inference, CUDA only)."""

    def __init__(self, input_size: int, output_size: int = 256, attention_heads: int = 4, linear_units: int = 2048, num_blocks: int = 6,
                 dropout_rate: float = 0.1, positional_dropout_rate: float = 0.1, attention_dropout_rate: float = 0.0,
                 input_layer: Optional[str] = "conv2d", pos_enc_class=None, pos_enc_layer_type: str = "abs_pos",
                 normalize_before: bool = True, concat_after: bool = False, positionwise_layer_type: str = "linear",
                 positionwise_conv_kernel_size: int = 1, padding_idx: int = -1, interctc_layer_idx: List[int] = [],
                 interctc_use_conditioning: bool = False, layer_drop_rate: float = 0.0, qk_norm: bool = False, use_flash_attn: bool = True):
        if (input_layer not in SUBSAMPLING or pos_enc_layer_type != "abs_pos" or not normalize_before or concat_after
                or positionwise_layer_type != "linear" or qk_norm):
            raise NotImplementedError("espnet_b200 TransformerEncoder: conv2d / conv2d2 / conv2d6 / conv2d8 input, abs_pos, pre-LN, linear feed-forward, no qk_norm")
        assert output_size % attention_heads == 0
        if output_size % 32:
            raise NotImplementedError("espnet_b200 TransformerEncoder: output_size must be a multiple of 32")
        super().__init__(input_size, output_size, (_Layer(output_size, linear_units) for _ in range(num_blocks)), input_layer)
        self.heads, self.num_blocks = attention_heads, num_blocks
        self._init_interctc(interctc_layer_idx, interctc_use_conditioning, num_blocks)
        self._pe = {}

    def _pack(self):
        pk = self._pack_io()
        pk["layers"] = [dict(n1=self._pack_ln(lyr.norm1), n2=self._pack_ln(lyr.norm2), **self._pack_mha(lyr.self_attn),
                             ffn=self._pack_ffn(lyr.feed_forward)) for lyr in self.encoders]
        self._packed = pk
        return pk

    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None, ctc=None):
        """xs_pad (B, T_f, idim) float32 CUDA, ilens (B,) -> (B, T, D), olens, None; per-utterance semantics for ragged batches.  With
        interctc_layer_idx the first element is ((B, T, D), [(layer, intermediate output), ...]) and, with interctc_use_conditioning, ctc is
        the CTC head (transformer_encoder.py:216-299)."""
        self._check_interctc(ctc)
        pk = self._packed or self._pack()
        xs_pad, T, olens, lens32 = self._lengths(xs_pad, ilens)   # check_short_utt: transformer_encoder.py:253-262
        B, D = xs_pad.shape[0], self._output_size
        M = B * T
        if T not in self._pe:
            if len(self._pe) > 8:
                self._pe.clear()
            self._pe[T] = abs_pos_table(T, D).to(xs_pad.device)

        # Conv2dSubsampling + PositionalEncoding: x = sqrt(D) * out(conv) + pe[t]
        x = self._buf("x", (M, D))
        self._subsample(xs_pad, x, math.sqrt(D), self._pe[T])
        if self.trace is not None:
            self.trace.append(x.view(B, T, D).clone())
        fused = ops.use_flash_attn(D // self.heads)   # one wgmma kernel for q k^T + masked softmax + p v (csrc/attention.cu)
        xn, qkv, ctx = self._buf("xn", (2, M, D)), self._buf("qkv", (2, M, 3 * D)), self._buf("ctx", (2, M, D))
        inter = []
        for li, w in enumerate(pk["layers"]):
            # x += MHA(LN1(x))  (encoder_layer.py:91-110, attention.py:262-265)
            layernorm(x, *w["n1"], LN_EPS, out_split=xn)
            linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
            self._attn(qkv, ctx, B, T, lens32, fused)
            linear(ctx, w["out_w"], x, bias=w["out_b"], residual=x)
            # x += w_2(relu(w_1(LN2(x))))  (encoder_layer.py:112-124)
            self._ffn(x, xn, w["n2"], w["ffn"], ACT_RELU, 1.0)
            if self.trace is not None:
                self.trace.append(x.view(B, T, D).clone())
            if li + 1 in self.interctc_layer_idx:
                inter.append((li + 1, self._interctc(x, B, T, ctc)))
        out, _ = self._output(x, B, T)
        return ((out, inter) if inter else out), olens, None
