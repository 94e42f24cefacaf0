"""ContextualBlockConformerEncoder and ContextualBlockTransformerEncoder: the streaming (block-synchronous) encoders of ESPnet2, many live
streams per call (SURVEY.md 8f-2, BASELINE configs[3]).

Reference: espnet2/asr/encoder/contextual_block_{conformer,transformer}_encoder.py (``forward_infer``: buffers before / after subsampling,
block framing with context tokens, output stitching -- the same code in both), legacy/nets/pytorch_backend/{conformer,transformer}/
contextual_block_encoder_layer.py (the layers and the context hand-over between blocks and layers), transformer/subsampling_without_posenc.py
(Conv2dSubsamplingWOPosEnc), transformer/embedding.py:337-388 (StreamPositionalEncoding).  Same constructor keywords / parameter names (a
reference checkpoint loads by name) and the same ``forward(xs_pad, ilens, prev_states, is_final, infer_mode=True) -> (ys_pad, olens,
next_states)`` protocol.

What differs: the reference asserts batch size 1 (one Python object per stream); here the batch dimension is a set of N live streams that push
equally long chunks in lock step, and all of their blocks run through the kernels together (N * blocks sequences of block_size + 2 tokens).
Only ``forward_infer`` exists (inference).  ``_ContextualBlockEncoder`` holds the streaming logic both encoders share; each encoder keeps its
constructor checks, its layer container, its packing and its per-layer sequence (``_layers``).  The subsampling (Conv2dSubsamplingWOPosEnc
has the parameters of Conv2dSubsampling{,6,8}), FFN, convolution module and masked self-attention are the shared ones of layers.py.
"""
import math
from typing import Optional, Tuple

import torch

from .layers import LN_EPS, MIN_FRAMES, SUBSAMPLING, EncoderBase, _ConvModule, _FFN, _MHA, abs_pos_table, subsampled_len
# gemm stays importable here although the shared code in layers.py launches the GEMMs: the kernel emulation of the tests replaces
# it in every encoder module
from .lib import call, ptr
from .ops import ACT_RELU, _count, gemm, layernorm, linear  # noqa: F401


class _ContextualBlockEncoder(EncoderBase):
    """forward_infer (contextual_block_conformer_encoder.py:386-600 = contextual_block_transformer_encoder.py:367-576) over N lock-step
    streams.  Subclasses define ``_pack`` and ``_layers``; ``has_olens`` says whether the final / short-utterance outputs come with lengths
    (the Conformer returns them, the Transformer returns None)."""

    has_olens = True

    def __init__(self, input_size, output_size, layers, input_layer, heads, num_blocks, block_size, hop_size, look_ahead):
        super().__init__(input_size, output_size, layers, input_layer)
        self.heads, self.num_blocks = heads, num_blocks
        self.block_size, self.hop_size, self.look_ahead = block_size, hop_size, look_ahead
        self.subsample = 2 * math.prod(s for _, s in SUBSAMPLING[input_layer])    # 4 / 6 / 8 for conv2d / conv2d6 / conv2d8
        self._pe = None

    def _pe_table(self, need):
        if self._pe is None or self._pe.shape[0] < need:
            self._pe = abs_pos_table(max(5000, 2 * need), self._output_size).to(self.after_norm.weight.device)
        return self._pe

    # ---------------------------------------------------------------- pieces of the per-layer sequences
    def _block_bufs(self, nseq, S, n_keys, zero_query0, N):
        """lens_k (n_keys keys per sequence), the xn / qkv / ctx workspaces and next_ctx [N][L][D] (None without zero_query0)."""
        D, L, M = self._output_size, self.num_blocks, nseq * S
        lens_k = self._buf("lens_k", (nseq,), dtype=torch.int32); lens_k.fill_(n_keys)
        xn, qkv, ctx = self._buf("xn", (2, M, D)), self._buf("qkv", (2, M, 3 * D)), self._buf("ctx", (2, M, D))
        next_ctx = torch.zeros(N, L, D, dtype=torch.float32, device=self._device) if zero_query0 else None
        return lens_k, xn, qkv, ctx, next_ctx

    def _self_attn(self, x, xn, qkv, ctx, w, nseq, S, lens_k, zero_query0):
        """x += linear_out(MHA(norm1(x))) over nseq sequences of S rows; keys 0..lens_k-1 are attended (the block mask lets tokens 1..S-1
        see tokens 0..S-2, contextual_block_conformer_encoder.py:543-549); zero_query0: token 0 attends nothing."""
        D, M = self._output_size, nseq * S
        layernorm(x, *w["norm1"], LN_EPS, out_split=xn)
        linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
        self._attn(qkv, ctx, nseq, S, lens_k, False)
        if zero_query0:   # the block mask has no key for token 0: its attention output is zero (masked_fill after the softmax)
            call("espb_zero_rows_f32", ptr(ctx), 0, S, nseq, D, M * D, 2)
            _count()
        linear(ctx, w["out_w"], x, bias=w["out_b"], residual=x)

    def _ctx_propagate(self, x, N, nb, S, past_ctx, next_ctx, li):
        """contextual_block_encoder_layer.py forward_infer, after the layer: token 0 of block i := last token of block i-1 (of block 0 or
        past_ctx for the first block); the last block's last token goes to next_ctx[:, li]."""
        call("espb_cbe_ctx_propagate_f32", ptr(x), N, nb, S, self._output_size, ptr(past_ctx), ptr(next_ctx), li, self.num_blocks)
        _count()

    # ---------------------------------------------------------------- forward_infer
    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states=None, is_final: bool = True, infer_mode: bool = True
                ) -> Tuple[torch.Tensor, Optional[torch.Tensor], Optional[dict]]:
        if not infer_mode:
            raise NotImplementedError(f"espnet_b200 {type(self).__name__} implements forward_infer only (infer_mode=True)")
        return self.forward_infer(xs_pad, ilens, prev_states, is_final)

    @torch.no_grad()
    def forward_infer(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states=None, is_final: bool = True):
        """xs_pad (N, L, idim): the next L feature frames of N live streams (all streams push the same L); prev_states: what the previous
        call returned (None for the first push); -> (ys_pad (N, T_out, D), olens (N,) or None, next_states | None)."""
        pk = self._packed or self._pack()
        st = prev_states or {}
        prev_addin, buf_before = st.get("prev_addin"), st.get("buffer_before_downsampling")
        buf_after, n_proc, past_ctx = st.get("buffer_after_downsampling"), st.get("n_processed_blocks", 0), st.get("past_encoder_ctx")
        xs_pad = xs_pad.contiguous().float()
        N, D = xs_pad.shape[0], self._output_size
        dev = xs_pad.device
        if buf_before is not None:
            xs_pad = torch.cat([buf_before, xs_pad], dim=1)

        def stash(**kw):
            base = dict(prev_addin=prev_addin, buffer_before_downsampling=buf_before, buffer_after_downsampling=buf_after,
                        n_processed_blocks=n_proc, past_encoder_ctx=past_ctx)
            base.update(kw)
            return base

        empty = lambda: (xs_pad.new_zeros(N, 0, D), xs_pad.new_zeros(N))  # noqa: E731
        if is_final:
            buf_before = None
        else:
            n_samples = xs_pad.shape[1] // self.subsample - 1
            if n_samples < 2:
                return (*empty(), stash(buffer_before_downsampling=xs_pad))
            n_res = xs_pad.shape[1] % self.subsample + self.subsample * 2
            buf_before = xs_pad[:, xs_pad.shape[1] - n_res:].contiguous()
            xs_pad = xs_pad[:, : n_samples * self.subsample].contiguous()
        if xs_pad.shape[1] >= MIN_FRAMES[self.input_layer]:   # Conv2dSubsamplingWOPosEnc: no scaling, no positional encoding
            xs = torch.empty(N, subsampled_len(xs_pad.shape[1], self.input_layer)[-1], D, dtype=torch.float32, device=dev)
            self._subsample(xs_pad, xs, 1.0)
        else:
            xs = xs_pad.new_zeros(N, 0, D)
        if buf_after is not None:
            xs = torch.cat([buf_after, xs], dim=1)
        total = xs.shape[1]
        B, Hp, LA = self.block_size, self.hop_size, self.look_ahead
        if is_final:
            past_size = B - Hp - LA
            block_num = math.ceil(float(total - past_size - LA) / float(Hp))
            buf_after = None
        else:
            if total <= B:
                return (*empty(), stash(buffer_before_downsampling=buf_before, buffer_after_downsampling=xs))
            overlap = B - Hp
            block_num = max(0, total - overlap) // Hp
            res = total - Hp * block_num
            buf_after = xs[:, total - res:].contiguous()
            xs = xs[:, : block_num * Hp + overlap].contiguous()
        pe = self._pe_table(Hp * (n_proc + block_num + 2) + B + 2)
        scale = math.sqrt(D)

        if n_proc == 0 and total <= B and is_final:
            # short utterance: the plain encoder over all frames, no context tokens (:479-488)
            x = torch.empty(N * total, D, dtype=torch.float32, device=dev)
            call("espb_cbe_build_chunks_f32", ptr(xs), N, total, D, 1, total, 1, ptr(pe), 0, 0, scale, None,
                 ptr(self._buf("addin_tmp", (N, D))), ptr(self._buf("short_chunk", (N, 1, total + 2, D))))
            _count()
            x.view(N, total, D).copy_(self._buf("short_chunk", (N, 1, total + 2, D))[:, 0, 1: total + 1])
            self._layers(x, N, total, pk, total, False, None, N, 1)
            out = torch.empty(N, total, D, dtype=torch.float32, device=dev)
            layernorm(x, *pk["after_norm"], LN_EPS, out_plain=out)
            return out, (xs_pad.new_zeros(N) if self.has_olens else None), None

        S = B + 2
        xs = xs.contiguous()
        chunks = torch.empty(N, block_num, S, D, dtype=torch.float32, device=dev)
        addin = torch.empty(N, D, dtype=torch.float32, device=dev)
        call("espb_cbe_build_chunks_f32", ptr(xs), N, xs.shape[1], D, block_num, B, Hp, ptr(pe), Hp * n_proc, n_proc, scale, ptr(prev_addin),
             ptr(addin), ptr(chunks))
        _count()
        next_ctx = self._layers(chunks.view(N * block_num * S, D), N * block_num, S, pk, B + 1, True, past_ctx, N, block_num)

        # stitch the outputs (:558-582): token r of block i is frame i*hop + (r - 1); the first `offset` frames of the stream come from
        # block 0, later frames from the block whose centre part covers them
        offset = B - LA - Hp
        if is_final:
            y_len = xs.shape[1] if n_proc == 0 else xs.shape[1] - offset
        else:
            y_len = block_num * Hp + (offset if n_proc == 0 else 0)
        idx = []
        if n_proc == 0:
            idx += [1 + t for t in range(offset)]
        for i in range(block_num):
            cur = i * Hp + (offset if n_proc == 0 else 0)
            n = min(B - offset, y_len - cur) if (i == block_num - 1 and is_final) else Hp
            idx += [i * S + 1 + offset + t for t in range(n)]
        assert len(idx) == y_len, (len(idx), y_len)
        idx_t = torch.tensor(idx, dtype=torch.int32, device=dev)
        ys = torch.empty(N, y_len, D, dtype=torch.float32, device=dev)
        call("espb_gather_rows_f32", ptr(chunks), N, block_num * S, ptr(idx_t), y_len, D, ptr(ys))
        _count()
        out = torch.empty_like(ys)
        layernorm(ys, *pk["after_norm"], LN_EPS, out_plain=out)
        olens = torch.full((N,), float(y_len), dtype=xs_pad.dtype, device=dev) if self.has_olens else None
        if is_final:
            return out, olens, None
        return out, olens, dict(prev_addin=addin, buffer_before_downsampling=buf_before, buffer_after_downsampling=buf_after,
                                n_processed_blocks=n_proc + block_num, past_encoder_ctx=next_ctx)


class _CBLayer(torch.nn.Module):
    def __init__(self, d, units, kernel, macaron):
        super().__init__()
        self.self_attn = _MHA(d)
        self.feed_forward = _FFN(d, units)
        self.feed_forward_macaron = _FFN(d, units) if macaron else None
        self.conv_module = _ConvModule(d, kernel)
        self.norm1 = torch.nn.LayerNorm(d, eps=LN_EPS)           # before the self-attention
        self.norm2 = torch.nn.LayerNorm(d, eps=LN_EPS)           # before the feed-forward
        if macaron:
            self.norm_ff_macaron = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_conv = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm_final = torch.nn.LayerNorm(d, eps=LN_EPS)


class ContextualBlockConformerEncoder(_ContextualBlockEncoder):
    """Supported configuration: input_layer "conv2d", normalize_before, cnn module, init_average, abs-pos self-attention (what
    ``ContextualBlockConformerEncoder`` builds), macaron optional."""

    def __init__(self, input_size: int, output_size: int = 256, attention_heads: int = 4, linear_units: int = 2048, num_blocks: int = 6,
                 dropout_rate: float = 0.1, positional_dropout_rate: float = 0.1, attention_dropout_rate: float = 0.0,
                 input_layer: Optional[str] = "conv2d", normalize_before: bool = True, concat_after: bool = False,
                 positionwise_layer_type: str = "linear", positionwise_conv_kernel_size: int = 3, macaron_style: bool = False,
                 pos_enc_class=None, selfattention_layer_type: str = "rel_selfattn", activation_type: str = "swish", use_cnn_module: bool = True,
                 cnn_module_kernel: int = 31, padding_idx: int = -1, block_size: int = 40, hop_size: int = 16, look_ahead: int = 16,
                 init_average: bool = True, ctx_pos_enc: bool = True):
        bad = []
        if input_layer != "conv2d": bad.append(f"input_layer={input_layer}")
        if not normalize_before or concat_after or not use_cnn_module: bad.append("non pre-LN / concat_after / no cnn module")
        if positionwise_layer_type != "linear" or activation_type != "swish": bad.append("positionwise / activation type")
        if not init_average or not ctx_pos_enc: bad.append("init_average / ctx_pos_enc = False")
        if block_size <= 0 or hop_size <= 0 or block_size - hop_size - look_ahead < 0: bad.append("block geometry")
        if cnn_module_kernel < 1 or cnn_module_kernel % 2 == 0 or cnn_module_kernel > 127:
            bad.append(f"cnn_module_kernel={cnn_module_kernel} (odd, <= 127)")
        if bad:
            raise NotImplementedError("espnet_b200 ContextualBlockConformerEncoder: " + ", ".join(bad))
        assert output_size % attention_heads == 0 and output_size % 32 == 0
        super().__init__(input_size, output_size,
                         (_CBLayer(output_size, linear_units, cnn_module_kernel, macaron_style) for _ in range(num_blocks)),
                         input_layer, attention_heads, num_blocks, block_size, hop_size, look_ahead)
        self.kernel, self.macaron = cnn_module_kernel, macaron_style

    def _pack(self):
        pk = self._pack_io()
        layers = []
        for lyr in self.encoders:
            d = {nm: self._pack_ln(getattr(lyr, nm)) for nm in ("norm1", "norm2", "norm_conv", "norm_final")}
            if self.macaron:
                d["norm_ff_macaron"], d["feed_forward_macaron"] = self._pack_ln(lyr.norm_ff_macaron), self._pack_ffn(lyr.feed_forward_macaron)
            d["feed_forward"] = self._pack_ffn(lyr.feed_forward)
            d.update(self._pack_mha(lyr.self_attn), **self._pack_conv(lyr.conv_module))
            layers.append(d)
        pk["layers"] = layers
        self._packed = pk
        return pk

    # ---------------------------------------------------------------- the layers over nseq sequences of S tokens
    def _layers(self, x, nseq, S, pk, n_keys, zero_query0, past_ctx, N, nb):
        """x [nseq*S][D] in place.  n_keys: keys 0..n_keys-1 of every sequence are attended; zero_query0: token 0 attends nothing.  Returns
        next_ctx [N][L][D] or None."""
        lens_k, xn, qkv, ctx, next_ctx = self._block_bufs(nseq, S, n_keys, zero_query0, N)
        lens_all = self._buf("lens_all", (nseq,), dtype=torch.int32); lens_all.fill_(S)
        ff_scale = 0.5 if self.macaron else 1.0
        # PositionwiseFeedForward's default ReLU: the encoder passes no activation (:163-168)
        for li, w in enumerate(pk["layers"]):
            if self.macaron:
                self._ffn(x, xn, w["norm_ff_macaron"], w["feed_forward_macaron"], ACT_RELU, ff_scale)
            self._self_attn(x, xn, qkv, ctx, w, nseq, S, lens_k, zero_query0)
            self._conv_module(x, xn, w["norm_conv"], w, nseq, S, lens_all)
            self._ffn(x, xn, w["norm2"], w["feed_forward"], ACT_RELU, ff_scale)
            layernorm(x, *w["norm_final"], LN_EPS, out_plain=x)
            if zero_query0:
                self._ctx_propagate(x, N, nb, S, past_ctx, next_ctx, li)
        return next_ctx


class _TBLayer(torch.nn.Module):
    """legacy/nets/pytorch_backend/transformer/contextual_block_encoder_layer.py: self_attn, feed_forward, norm1, norm2."""

    def __init__(self, d, units):
        super().__init__()
        self.self_attn = _MHA(d)
        self.feed_forward = _FFN(d, units)
        self.norm1 = torch.nn.LayerNorm(d, eps=LN_EPS)           # before the self-attention
        self.norm2 = torch.nn.LayerNorm(d, eps=LN_EPS)           # before the feed-forward


class ContextualBlockTransformerEncoder(_ContextualBlockEncoder):
    """espnet2/asr/encoder/contextual_block_transformer_encoder.py (Tsunoo et al., arXiv:1910.07204).  Each layer is norm1 -> self-attention
    -> residual, norm2 -> ReLU feed-forward -> residual.  Supported configuration: input_layer "conv2d" / "conv2d6" / "conv2d8",
    normalize_before, linear feed-forward, init_average, ctx_pos_enc; ``forward_infer`` returns no lengths (olens None), as the reference."""

    has_olens = False

    def __init__(self, input_size: int, output_size: int = 256, attention_heads: int = 4, linear_units: int = 2048, num_blocks: int = 6,
                 dropout_rate: float = 0.1, positional_dropout_rate: float = 0.1, attention_dropout_rate: float = 0.0,
                 input_layer: Optional[str] = "conv2d", pos_enc_class=None, normalize_before: bool = True, concat_after: bool = False,
                 positionwise_layer_type: str = "linear", positionwise_conv_kernel_size: int = 1, padding_idx: int = -1,
                 block_size: int = 40, hop_size: int = 16, look_ahead: int = 16, init_average: bool = True, ctx_pos_enc: bool = True):
        if input_layer not in ("conv2d", "conv2d6", "conv2d8", "linear", "embed", None):
            raise ValueError(f"unknown input_layer: {input_layer}")
        bad = []
        if input_layer not in ("conv2d", "conv2d6", "conv2d8"): bad.append(f"input_layer={input_layer}")
        if pos_enc_class is not None and getattr(pos_enc_class, "__name__", None) != "StreamPositionalEncoding": bad.append("pos_enc_class")
        if not normalize_before or concat_after: bad.append("non pre-LN / concat_after")
        if positionwise_layer_type != "linear": bad.append(f"positionwise_layer_type={positionwise_layer_type}")
        if not init_average or not ctx_pos_enc: bad.append("init_average / ctx_pos_enc = False")
        if output_size % 32: bad.append("output_size not a multiple of 32")
        if block_size <= 0 or hop_size <= 0 or block_size - hop_size - look_ahead < 0: bad.append("block geometry")
        if bad:
            raise NotImplementedError("espnet_b200 ContextualBlockTransformerEncoder: " + ", ".join(bad))
        assert output_size % attention_heads == 0
        super().__init__(input_size, output_size, (_TBLayer(output_size, linear_units) for _ in range(num_blocks)), input_layer,
                         attention_heads, num_blocks, block_size, hop_size, look_ahead)

    def _pack(self):
        pk = self._pack_io()
        pk["layers"] = [dict(norm1=self._pack_ln(lyr.norm1), norm2=self._pack_ln(lyr.norm2), feed_forward=self._pack_ffn(lyr.feed_forward),
                             **self._pack_mha(lyr.self_attn)) for lyr in self.encoders]
        self._packed = pk
        return pk

    def _layers(self, x, nseq, S, pk, n_keys, zero_query0, past_ctx, N, nb):
        """As ContextualBlockConformerEncoder._layers, with the Transformer layer: self-attention, then the ReLU feed-forward (ff_scale 1)."""
        lens_k, xn, qkv, ctx, next_ctx = self._block_bufs(nseq, S, n_keys, zero_query0, N)
        for li, w in enumerate(pk["layers"]):
            self._self_attn(x, xn, qkv, ctx, w, nseq, S, lens_k, zero_query0)
            self._ffn(x, xn, w["norm2"], w["feed_forward"], ACT_RELU, 1.0)
            if zero_query0:
                self._ctx_propagate(x, N, nb, S, past_ctx, next_ctx, li)
        return next_ctx
