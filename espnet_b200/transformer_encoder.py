"""TransformerEncoder (absolute positions, conv2d input layer, pre-LN, ReLU feed-forward) with the reference's constructor /
state_dict surface -- the encoder of the next scope row (SURVEY.md 8f-1, BASELINE configs[4]).  It composes the kernels of the
Conformer path (conv1 / implicit-GEMM conv2 / wgmma 3xTF32 GEMMs / LayerNorm) plus a plain masked softmax.

Reference: espnet2/asr/encoder/transformer_encoder.py:43-299, legacy/nets/pytorch_backend/transformer/encoder_layer.py:65-126,
attention.py:77-151,262-265 (default branch), embedding.py:38-95 (PositionalEncoding), subsampling.py:397-474.
Parity: tests/test_gpu_zz_next.py (reference fixture layer by layer, ragged batch, whole Speech2Text) and tests/test_host_logic_emulated.py; self-attention
is the fused wgmma kernel without the rel-pos term (csrc/attention.cu) at d_k = 64.
"""
import math
from typing import List, Optional, Tuple

import torch

from . import ops
from .encoder import LN_EPS, _Conv2dSubsampling, _FFN
from .errors import TooShortUttError
from .lib import call, ptr
from .ops import ACT_RELU, _count, gemm, layernorm, linear, split_from


class _MHA(torch.nn.Module):
    def __init__(self, n_feat):
        super().__init__()
        self.linear_q = torch.nn.Linear(n_feat, n_feat)
        self.linear_k = torch.nn.Linear(n_feat, n_feat)
        self.linear_v = torch.nn.Linear(n_feat, n_feat)
        self.linear_out = torch.nn.Linear(n_feat, n_feat)


class _Layer(torch.nn.Module):
    def __init__(self, d, units):
        super().__init__()
        self.self_attn = _MHA(d)
        self.feed_forward = _FFN(d, units)
        self.norm1 = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm2 = torch.nn.LayerNorm(d, eps=LN_EPS)


def abs_pos_table(T, d):
    """PositionalEncoding.extend_pe (embedding.py:62-83)."""
    pos = torch.arange(0, T, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe = torch.zeros(T, d)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


class TransformerEncoder(torch.nn.Module):
    """Drop-in for espnet2.asr.encoder.transformer_encoder.TransformerEncoder (inference, CUDA only)."""

    def __init__(self, input_size: int, output_size: int = 256, attention_heads: int = 4, linear_units: int = 2048, num_blocks: int = 6,
                 dropout_rate: float = 0.1, positional_dropout_rate: float = 0.1, attention_dropout_rate: float = 0.0,
                 input_layer: Optional[str] = "conv2d", pos_enc_class=None, pos_enc_layer_type: str = "abs_pos",
                 normalize_before: bool = True, concat_after: bool = False, positionwise_layer_type: str = "linear",
                 positionwise_conv_kernel_size: int = 1, padding_idx: int = -1, interctc_layer_idx: List[int] = [],
                 interctc_use_conditioning: bool = False, layer_drop_rate: float = 0.0, qk_norm: bool = False, use_flash_attn: bool = True):
        super().__init__()
        if (input_layer != "conv2d" or pos_enc_layer_type != "abs_pos" or not normalize_before or concat_after
                or positionwise_layer_type != "linear" or qk_norm or len(interctc_layer_idx)):
            raise NotImplementedError("espnet_b200 TransformerEncoder: conv2d input, abs_pos, pre-LN, linear feed-forward, no interCTC / qk_norm")
        assert output_size % attention_heads == 0
        if output_size % 32:
            raise NotImplementedError("espnet_b200 TransformerEncoder: output_size must be a multiple of 32")
        self._output_size, self.heads, self.units, self.num_blocks, self.idim = output_size, attention_heads, linear_units, num_blocks, input_size
        self.embed = _Conv2dSubsampling(input_size, output_size)
        self.encoders = torch.nn.ModuleList(_Layer(output_size, linear_units) for _ in range(num_blocks))
        self.after_norm = torch.nn.LayerNorm(output_size, eps=LN_EPS)
        self._packed, self._ws, self._pe = None, {}, {}
        self.trace = None
        self.last_split_out = None

    def output_size(self) -> int:
        return self._output_size

    def _load_from_state_dict(self, *args, **kwargs):
        self._packed = None
        return super()._load_from_state_dict(*args, **kwargs)

    def _pack(self):
        dev = self.after_norm.weight.device
        D = C = self._output_size
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        e = self.embed
        F1 = (self.idim - 3) // 2 + 1
        F2 = (F1 - 3) // 2 + 1
        pk = dict(F1=F1, F2=F2, c1_w=f32(e.conv[0].weight).view(C, 9), c1_b=f32(e.conv[0].bias),
                  c2_w=split_from(f32(e.conv[2].weight).permute(0, 2, 3, 1).reshape(C, 9 * C)), c2_b=f32(e.conv[2].bias),
                  # embed.out columns are c*F2+f (subsampling.py:450-451) -> f*C+c to match the [B][F2][T][C] conv2 output
                  out_w=split_from(f32(e.out.weight).view(D, C, F2).permute(0, 2, 1).reshape(D, F2 * C)), out_b=f32(e.out.bias), layers=[])
        for lyr in self.encoders:
            a, ff = lyr.self_attn, lyr.feed_forward
            pk["layers"].append(dict(
                n1=(f32(lyr.norm1.weight), f32(lyr.norm1.bias)), n2=(f32(lyr.norm2.weight), f32(lyr.norm2.bias)),
                qkv_w=split_from(torch.cat([f32(a.linear_q.weight), f32(a.linear_k.weight), f32(a.linear_v.weight)], 0)),
                qkv_b=torch.cat([f32(a.linear_q.bias), f32(a.linear_k.bias), f32(a.linear_v.bias)], 0),
                out_w=split_from(f32(a.linear_out.weight)), out_b=f32(a.linear_out.bias),
                w1=split_from(f32(ff.w_1.weight)), b1=f32(ff.w_1.bias), w2=split_from(f32(ff.w_2.weight)), b2=f32(ff.w_2.bias)))
        pk["after_norm"] = (f32(self.after_norm.weight), f32(self.after_norm.bias))
        self._packed = pk
        return pk

    def _buf(self, name, shape, zero=False):
        key = (name, tuple(shape))
        t = self._ws.get(key)
        if t is None:
            t = (torch.zeros if zero else torch.empty)(shape, dtype=torch.float32, device=self.after_norm.weight.device)
            for k in [k for k in self._ws if k[0] == name and k != key]:
                del self._ws[k]
            self._ws[key] = t
        return t

    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """xs_pad (B, T_f, idim) float32 CUDA, ilens (B,) -> (B, T, D), olens, None; per-utterance semantics for ragged batches."""
        pk = self._packed or self._pack()
        dev = xs_pad.device
        xs_pad = xs_pad.contiguous().float()
        B, Tf, F = xs_pad.shape
        assert F == self.idim
        # check_short_utt (subsampling.py:43-44), transformer_encoder.py:253-262: the reference decodes one utterance per call, so the limit applies to every
        # utterance of a ragged batch, not to the padded length (an utterance with < 7 frames would get olens 0)
        min_len = int(torch.as_tensor(ilens).min()) if torch.as_tensor(ilens).numel() else Tf
        if Tf < 7 or min_len < 7:
            size = min(Tf, min_len)
            which = "" if Tf < 7 else f" (utterance {int(torch.as_tensor(ilens).argmin())} of the batch)"
            raise TooShortUttError(f"has {size} frames and is too short for subsampling (it needs more than 7 frames), "
                                   f"return empty results{which}", size, 7)
        D, H, U = self._output_size, self.heads, self.units
        C, dk = D, D // H
        F1, F2 = pk["F1"], pk["F2"]
        T1 = (Tf - 3) // 2 + 1
        T = (T1 - 3) // 2 + 1
        T1h, F1h = (T1 + 1) // 2, (F1 + 1) // 2
        olens = torch.div(torch.div(ilens - 1, 2, rounding_mode="trunc") - 1, 2, rounding_mode="trunc")
        lens32 = olens.to(device=dev, dtype=torch.int32).contiguous()
        M = B * T
        Tp = (T + 31) // 32 * 32
        if T not in self._pe:
            if len(self._pe) > 8:
                self._pe.clear()
            self._pe[T] = abs_pos_table(T, D).to(dev)

        # ---- Conv2dSubsampling + PositionalEncoding: x = sqrt(D) * out(conv) + pe[t]  (the table enters as a batch-broadcast residual)
        c1 = self._buf("c1", (B, 8, F1h, T1h, C), zero=True)
        call("espb_conv1_relu_f32", ptr(xs_pad), B, Tf, F, ptr(pk["c1_w"]), ptr(pk["c1_b"]), C, ptr(c1), T1, F1, T1h, F1h)
        _count()
        c2 = self._buf("c2", (2, B, F2, T, C))
        gemm(T, C, 9 * C, c1, 0, 0, pk["c2_w"], C * 9 * C, 9 * C, c2, C, c_plane=B * F2 * T * C, split_out=True, bias=pk["c2_b"],
             act=ACT_RELU, nbx=F2, nby=B, sc=(T * C, F2 * T * C), a_mode=1, conv=(T1h, F1h, C))
        x = self._buf("x", (M, D))
        gemm(T, D, F2 * C, c2, B * F2 * T * C, C, pk["out_w"], D * F2 * C, F2 * C, x, D, bias=pk["out_b"], alpha=math.sqrt(D),
             R=self._pe[T], ldr=D, sr=(0, 0), nbx=1, nby=B, sa=(T * C, F2 * T * C), sc=(0, T * D), kob=C // 32)
        if self.trace is not None:
            self.trace.append(x.view(B, T, D).clone())

        xn = self._buf("xn", (2, M, D))
        hbuf = self._buf("h", (2, M, U))
        qkv = self._buf("qkv", (2, M, 3 * D))
        vt = self._buf("vt", (2, B, H, dk, Tp))
        fused = ops.use_flash_attn(dk)      # one wgmma kernel for q k^T + masked softmax + p v (csrc/attention.cu)
        if not fused:
            sc = self._buf("sc", (B, H, T, Tp))
            probs = self._buf("probs", (2, B, H, T, Tp))
        ctx = self._buf("ctx", (2, M, D))
        for w in pk["layers"]:
            # x += MHA(LN1(x))  (encoder_layer.py:91-110, attention.py:262-265)
            layernorm(x, *w["n1"], LN_EPS, out_split=xn)
            linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
            call("espb_v_transpose_f32", ptr(qkv), M * 3 * D, B, T, D, H, ptr(lens32), ptr(vt), B * H * dk * Tp, Tp)
            _count()
            if fused:
                ops.flash_attn(qkv, 0, 3 * D, qkv, D, 3 * D, vt, Tp, None, 0, lens32, B, H, T, dk, ctx)
            else:
                gemm(T, T, dk, qkv, M * 3 * D, 3 * D, qkv, M * 3 * D, 3 * D, sc, Tp, nbx=H, nby=B, sa=(dk, T * 3 * D), sb=(dk, T * 3 * D),
                     sc=(T * Tp, H * T * Tp), b_off=D)
                call("espb_masked_softmax_f32", ptr(sc), B, H, T, Tp, ptr(lens32), math.sqrt(dk), ptr(probs), B * H * T * Tp)
                _count()
                gemm(T, dk, T, probs, B * H * T * Tp, Tp, vt, B * H * dk * Tp, Tp, ctx, D, c_plane=M * D, split_out=True, nbx=H, nby=B,
                     sa=(T * Tp, H * T * Tp), sb=(dk * Tp, H * dk * Tp), sc=(dk, T * D))
            linear(ctx, w["out_w"], x, bias=w["out_b"], residual=x)
            # x += w_2(relu(w_1(LN2(x))))  (encoder_layer.py:112-124)
            layernorm(x, *w["n2"], LN_EPS, out_split=xn)
            linear(xn, w["w1"], hbuf, bias=w["b1"], act=ACT_RELU, split_out=True)
            linear(hbuf, w["w2"], x, bias=w["b2"], residual=x)
            if self.trace is not None:
                self.trace.append(x.view(B, T, D).clone())
        out = torch.empty(B, T, D, dtype=torch.float32, device=dev)
        out_split = self._buf("enc_split", (2, M, D))
        layernorm(x, *pk["after_norm"], LN_EPS, out_plain=out, out_split=out_split)
        self.last_split_out = (out.data_ptr(), out_split)
        return out, olens, None
