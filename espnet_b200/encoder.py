"""ConformerEncoder with the reference's constructor / state_dict surface, executed by the espnet_b200
CUDA kernels (wgmma 3xTF32 GEMMs + warp-primitive glue).

Reference: espnet2/asr/encoder/conformer_encoder.py:89-429 and the legacy modules it composes
(Conv2dSubsampling, RelPositionalEncoding, EncoderLayer, RelPositionMultiHeadedAttention,
PositionwiseFeedForward, ConvolutionModule, LayerNorm).  Supported configuration = the one
BASELINE.json names: input_layer "conv2d", rel_pos_type "latest" (rel_pos / rel_selfattn),
macaron_style, use_cnn_module, swish, normalize_before, no intermediate CTC.  The torch.nn layers
below are parameter containers only (so that reference checkpoints load by name); forward never
calls them.
"""
import math
from typing import List, Optional, Tuple, Union

import torch

from . import ops
from .errors import TooShortUttError
from .lib import call, ptr
from .ops import ACT_NONE, ACT_RELU, ACT_SWISH, _count, gemm, layernorm, linear, new_split, split_from

LN_EPS = 1e-12  # transformer/layer_norm.py:22


class _PosBias(torch.nn.Module):
    def __init__(self, n_head, n_feat):
        super().__init__()
        d_k = n_feat // n_head
        self.linear_q = torch.nn.Linear(n_feat, n_feat)
        self.linear_k = torch.nn.Linear(n_feat, n_feat)
        self.linear_v = torch.nn.Linear(n_feat, n_feat)
        self.linear_out = torch.nn.Linear(n_feat, n_feat)
        self.linear_pos = torch.nn.Linear(n_feat, n_feat, bias=False)
        self.pos_bias_u = torch.nn.Parameter(torch.Tensor(n_head, d_k))
        self.pos_bias_v = torch.nn.Parameter(torch.Tensor(n_head, d_k))
        torch.nn.init.xavier_uniform_(self.pos_bias_u)
        torch.nn.init.xavier_uniform_(self.pos_bias_v)


class _FFN(torch.nn.Module):
    def __init__(self, d, units):
        super().__init__()
        self.w_1 = torch.nn.Linear(d, units)
        self.w_2 = torch.nn.Linear(units, d)


class _ConvModule(torch.nn.Module):
    def __init__(self, channels, kernel_size):
        super().__init__()
        assert (kernel_size - 1) % 2 == 0
        self.pointwise_conv1 = torch.nn.Conv1d(channels, 2 * channels, 1)
        self.depthwise_conv = torch.nn.Conv1d(channels, channels, kernel_size, padding=(kernel_size - 1) // 2, groups=channels)
        self.norm = torch.nn.BatchNorm1d(channels)
        self.pointwise_conv2 = torch.nn.Conv1d(channels, channels, 1)


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


class _Conv2dSubsampling(torch.nn.Module):
    def __init__(self, idim, odim):
        super().__init__()
        self.conv = torch.nn.Sequential(torch.nn.Conv2d(1, odim, 3, 2), torch.nn.ReLU(), torch.nn.Conv2d(odim, odim, 3, 2),
                                        torch.nn.ReLU())
        self.out = torch.nn.Linear(odim * (((idim - 1) // 2 - 1) // 2), odim)


def rel_pos_table(T, d):
    """(2T-1, d) slice RelPositionalEncoding.forward returns: row k = sinusoid of relative position T-1-k
    (embedding.py:286-334).  Built once per length on the host, like the reference's ``pe`` buffer."""
    pos = torch.arange(T - 1, -T, -1, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe = torch.zeros(2 * T - 1, d)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


class ConformerEncoder(torch.nn.Module):
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
        super().__init__()
        unsupported = []
        if input_layer != "conv2d": unsupported.append(f"input_layer={input_layer}")
        if rel_pos_type != "latest" or pos_enc_layer_type != "rel_pos" or selfattention_layer_type != "rel_selfattn":
            unsupported.append("rel_pos_type/pos_enc_layer_type/selfattention_layer_type other than latest/rel_pos/rel_selfattn")
        if not (normalize_before and macaron_style and use_cnn_module) or concat_after: unsupported.append("non pre-LN macaron+cnn block")
        if positionwise_layer_type != "linear" or activation_type != "swish": unsupported.append("positionwise/activation type")
        if zero_triu or qk_norm or len(interctc_layer_idx) or ctc_trim: unsupported.append("zero_triu/qk_norm/interctc/ctc_trim")
        if unsupported:
            raise NotImplementedError("espnet_b200 ConformerEncoder supports the BASELINE configuration only; got " + ", ".join(unsupported))
        assert output_size % attention_heads == 0
        if output_size % 32:
            raise NotImplementedError("espnet_b200 ConformerEncoder: output_size must be a multiple of 32")
        self._output_size, self.heads, self.units, self.num_blocks = output_size, attention_heads, linear_units, num_blocks
        self.kernel, self.idim = cnn_module_kernel, input_size
        self.embed = _Conv2dSubsampling(input_size, output_size)
        self.encoders = torch.nn.ModuleList(_EncoderLayer(output_size, attention_heads, linear_units, cnn_module_kernel)
                                            for _ in range(num_blocks))
        self.after_norm = torch.nn.LayerNorm(output_size, eps=LN_EPS)
        self._packed = None
        self._ws = {}
        self._pos_cache = {}
        self.trace = None  # set to a list to collect per-stage outputs (tests)
        self.last_split_out = None  # split copy of the last output (feeds the CTC head / decoder memory GEMMs)

    def output_size(self) -> int:
        return self._output_size

    # ---------------------------------------------------------------- weights -> device-side packed/split form
    def _load_from_state_dict(self, *args, **kwargs):
        self._packed = None
        return super()._load_from_state_dict(*args, **kwargs)

    def invalidate(self):
        self._packed = None

    def _pack(self):
        dev = self.after_norm.weight.device
        D, C = self._output_size, self._output_size
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        e = self.embed
        F1 = (self.idim - 3) // 2 + 1
        F2 = (F1 - 3) // 2 + 1
        pk = dict(F1=F1, F2=F2)
        pk["c1_w"] = f32(e.conv[0].weight).view(C, 9)
        pk["c1_b"] = f32(e.conv[0].bias)
        # conv2 weight [co][ci][kt][kf] -> [co][(kt*3+kf)*C + ci]
        pk["c2_w"] = split_from(f32(e.conv[2].weight).permute(0, 2, 3, 1).reshape(C, 9 * C))
        pk["c2_b"] = f32(e.conv[2].bias)
        # embed.out columns are c*F2+f (subsampling.py:450-451) -> f*C+c to match the [B][F2][T][C] conv2 output
        pk["out_w"] = split_from(f32(e.out.weight).view(D, C, F2).permute(0, 2, 1).reshape(D, F2 * C))
        pk["out_b"] = f32(e.out.bias)
        layers = []
        for lyr in self.encoders:
            a, cm = lyr.self_attn, lyr.conv_module
            d = {}
            for nm in ("norm_ff_macaron", "norm_mha", "norm_conv", "norm_ff", "norm_final"):
                m = getattr(lyr, nm)
                d[nm] = (f32(m.weight), f32(m.bias))
            for nm in ("feed_forward_macaron", "feed_forward"):
                m = getattr(lyr, nm)
                d[nm] = (split_from(f32(m.w_1.weight)), f32(m.w_1.bias), split_from(f32(m.w_2.weight)), f32(m.w_2.bias))
            d["qkv_w"] = split_from(torch.cat([f32(a.linear_q.weight), f32(a.linear_k.weight), f32(a.linear_v.weight)], 0))
            d["qkv_b"] = torch.cat([f32(a.linear_q.bias), f32(a.linear_k.bias), f32(a.linear_v.bias)], 0)
            d["out_w"], d["out_b"] = split_from(f32(a.linear_out.weight)), f32(a.linear_out.bias)
            d["pos_u"], d["pos_v"] = f32(a.pos_bias_u).view(-1), f32(a.pos_bias_v).view(-1)
            d["pw1_w"], d["pw1_b"] = split_from(f32(cm.pointwise_conv1.weight).view(2 * D, D)), f32(cm.pointwise_conv1.bias)
            d["dw_w"], d["dw_b"] = f32(cm.depthwise_conv.weight).view(D, -1), f32(cm.depthwise_conv.bias)
            # BatchNorm1d eval: y = x*alpha + beta with alpha = weight/sqrt(var+eps) (what ATen's CPU kernel computes)
            inv = 1.0 / torch.sqrt(f32(cm.norm.running_var) + cm.norm.eps)
            alpha = inv * f32(cm.norm.weight)
            d["bn_a"], d["bn_b"] = alpha.contiguous(), (f32(cm.norm.bias) - f32(cm.norm.running_mean) * alpha).contiguous()
            d["pw2_w"], d["pw2_b"] = split_from(f32(cm.pointwise_conv2.weight).view(D, D)), f32(cm.pointwise_conv2.bias)
            layers.append(d)
        pk["layers"] = layers
        pk["pos_w_all"] = split_from(torch.cat([f32(l.self_attn.linear_pos.weight) for l in self.encoders], 0))  # [L*D][D]
        pk["after_norm"] = (f32(self.after_norm.weight), f32(self.after_norm.bias))
        self._packed = pk
        return pk

    def _buf(self, name, shape, zero=False):
        key = (name, tuple(shape))
        t = self._ws.get(key)
        if t is None:
            dev = self.after_norm.weight.device
            t = (torch.zeros if zero else torch.empty)(shape, dtype=torch.float32, device=dev)
            # drop stale buffers of the same name with other shapes
            for k in [k for k in self._ws if k[0] == name and k != key]:
                del self._ws[k]
            self._ws[key] = t
        return t

    def _pos(self, T, pk):
        """P_all split [2][2T-1][L*D] = linear_pos(pos_emb) for every layer (one GEMM per length, cached)."""
        if T not in self._pos_cache:
            if len(self._pos_cache) > 8:
                self._pos_cache.clear()
            D, L = self._output_size, self.num_blocks
            pe = split_from(rel_pos_table(T, D).to(self.after_norm.weight.device))
            out = new_split(2 * T - 1, L * D, device=pe.device)
            linear(pe, pk["pos_w_all"], out, split_out=True)
            self._pos_cache[T] = out
        return self._pos_cache[T]

    # ---------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """xs_pad (B, T_f, idim) float32 CUDA (normalised log-mel), ilens (B,) -> (B, T, D), olens, None.

        Ragged batches follow per-utterance (batch-1) semantics of the reference: every utterance sees only
        its own frames (own conv boundaries, own attention keys); rows t >= olens[b] of the output are padding."""
        pk = self._packed or self._pack()
        dev = xs_pad.device
        xs_pad = xs_pad.contiguous().float()
        B, Tf, F = xs_pad.shape
        assert F == self.idim
        # check_short_utt (subsampling.py:43-44), conformer_encoder.py:363-371: the reference decodes one utterance per call, so the limit applies to every
        # utterance of a ragged batch, not to the padded length (an utterance with < 7 frames would get olens 0)
        min_len = int(torch.as_tensor(ilens).min()) if torch.as_tensor(ilens).numel() else Tf
        if Tf < 7 or min_len < 7:
            size = min(Tf, min_len)
            which = "" if Tf < 7 else f" (utterance {int(torch.as_tensor(ilens).argmin())} of the batch)"
            raise TooShortUttError(f"has {size} frames and is too short for subsampling (it needs more than 7 frames), "
                                   f"return empty results{which}", size, 7)
        D, H, L, U, K = self._output_size, self.heads, self.num_blocks, self.units, self.kernel
        C, dk = D, D // H
        F1, F2 = pk["F1"], pk["F2"]
        T1 = (Tf - 3) // 2 + 1
        T = (T1 - 3) // 2 + 1
        T1h, F1h = (T1 + 1) // 2, (F1 + 1) // 2
        olens = torch.div(torch.div(ilens - 1, 2, rounding_mode="trunc") - 1, 2, rounding_mode="trunc")
        lens32 = olens.to(device=dev, dtype=torch.int32).contiguous()
        M = B * T
        # row pitches of the score / probability matrices: multiples of 32 floats so that every 128-byte store segment of the GEMM
        # epilogues is a whole cache line (partial-sector writes cost a DRAM read-modify-write)
        Tp, Rp = (T + 31) // 32 * 32, (2 * T - 1 + 31) // 32 * 32

        # ---- Conv2dSubsampling (subsampling.py:432-474)
        c1 = self._buf("c1", (B, 8, F1h, T1h, C), zero=True)
        call("espb_conv1_relu_f32", ptr(xs_pad), B, Tf, F, ptr(pk["c1_w"]), ptr(pk["c1_b"]), C, ptr(c1), T1, F1, T1h, F1h)
        _count()
        c2 = self._buf("c2", (2, B, F2, T, C))
        gemm(T, C, 9 * C, c1, 0, 0, pk["c2_w"], C * 9 * C, 9 * C, c2, C, c_plane=B * F2 * T * C, split_out=True, bias=pk["c2_b"],
             act=ACT_RELU, nbx=F2, nby=B, sc=(T * C, F2 * T * C), a_mode=1, conv=(T1h, F1h, C))
        x = self._buf("x", (M, D))
        gemm(T, D, F2 * C, c2, B * F2 * T * C, C, pk["out_w"], D * F2 * C, F2 * C, x, D, bias=pk["out_b"], alpha=math.sqrt(D),
             nbx=1, nby=B, sa=(T * C, F2 * T * C), sc=(0, T * D), kob=C // 32)
        if self.trace is not None:
            self.trace.append(x.view(B, T, D).clone())
        p_all = self._pos(T, pk)
        R = 2 * T - 1

        xn = self._buf("xn", (2, M, D))
        hbuf = self._buf("h", (2, M, U))
        qkv = self._buf("qkv", (2, M, 3 * D))
        qu, qv = self._buf("qu", (2, M, D)), self._buf("qv", (2, M, D))
        vt = self._buf("vt", (2, B, H, dk, Tp))
        bd = self._buf("bd", (B, H, T, Rp))
        fused = ops.use_flash_attn(dk)      # one wgmma kernel for q k^T + rel_shift + softmax + p v (csrc/attention.cu); else materialised
        if not fused:
            ac = self._buf("ac", (B, H, T, Tp))
            probs = self._buf("probs", (2, B, H, T, Tp))
        ctx = self._buf("ctx", (2, M, D))
        y = self._buf("y", (M, 2 * D))
        cv = self._buf("cv", (2, M, D))
        for li, w in enumerate(pk["layers"]):
            # macaron FFN: x += 0.5 * w2(swish(w1(LN(x))))   (encoder_layer.py:115-123)
            w1, b1, w2, b2 = w["feed_forward_macaron"]
            layernorm(x, *w["norm_ff_macaron"], LN_EPS, out_split=xn)
            linear(xn, w1, hbuf, bias=b1, act=ACT_SWISH, split_out=True)
            linear(hbuf, w2, x, bias=b2, residual=x, alpha=0.5)
            # rel-pos MHSA (encoder_layer.py:126-149, attention.py:416-459)
            layernorm(x, *w["norm_mha"], LN_EPS, out_split=xn)
            linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
            call("espb_qu_qv_f32", ptr(qkv), M * 3 * D, M, D, ptr(w["pos_u"]), ptr(w["pos_v"]), ptr(qu), ptr(qv), M * D)
            call("espb_v_transpose_f32", ptr(qkv), M * 3 * D, B, T, D, H, ptr(lens32), ptr(vt), B * H * dk * Tp, Tp)
            _count(2)
            gemm(T, R, dk, qv, M * D, D, p_all, R * L * D, L * D, bd, Rp, nbx=H, nby=B, sa=(dk, T * D), sb=(dk, 0),
                 sc=(T * Rp, H * T * Rp), b_off=li * D, band_t=T)   # rel_shift only ever reads bd[i][T-1-i .. 2T-2-i]
            if fused:
                ops.flash_attn(qu, 0, D, qkv, D, 3 * D, vt, Tp, bd, Rp, lens32, B, H, T, dk, ctx)
            else:
                gemm(T, T, dk, qu, M * D, D, qkv, M * 3 * D, 3 * D, ac, Tp, nbx=H, nby=B, sa=(dk, T * D), sb=(dk, T * 3 * D),
                     sc=(T * Tp, H * T * Tp), b_off=D)
                call("espb_relpos_softmax_f32", ptr(ac), ptr(bd), B, H, T, Tp, Rp, ptr(lens32), math.sqrt(dk), ptr(probs), B * H * T * Tp)
                _count()
                gemm(T, dk, T, probs, B * H * T * Tp, Tp, vt, B * H * dk * Tp, Tp, ctx, D, c_plane=M * D, split_out=True, nbx=H, nby=B,
                     sa=(T * Tp, H * T * Tp), sb=(dk * Tp, H * dk * Tp), sc=(dk, T * D))
            linear(ctx, w["out_w"], x, bias=w["out_b"], residual=x)
            # convolution module (encoder_layer.py:152-158, convolution.py:56-79)
            layernorm(x, *w["norm_conv"], LN_EPS, out_split=xn)
            linear(xn, w["pw1_w"], y, bias=w["pw1_b"])
            call("espb_glu_dwconv_bn_swish_f32", ptr(y), B, T, D, ptr(lens32), ptr(w["dw_w"]), ptr(w["dw_b"]), K, ptr(w["bn_a"]),
                 ptr(w["bn_b"]), ptr(cv), M * D)
            _count()
            linear(cv, w["pw2_w"], x, bias=w["pw2_b"], residual=x)
            # FFN + final norm (encoder_layer.py:161-171)
            w1, b1, w2, b2 = w["feed_forward"]
            layernorm(x, *w["norm_ff"], LN_EPS, out_split=xn)
            linear(xn, w1, hbuf, bias=b1, act=ACT_SWISH, split_out=True)
            linear(hbuf, w2, x, bias=b2, residual=x, alpha=0.5)
            layernorm(x, *w["norm_final"], LN_EPS, out_plain=x)
            if self.trace is not None:
                self.trace.append(x.view(B, T, D).clone())
        out = torch.empty(B, T, D, dtype=torch.float32, device=dev)
        out_split = self._buf("enc_split", (2, M, D))
        layernorm(x, *pk["after_norm"], LN_EPS, out_plain=out, out_split=out_split)
        self.last_split_out = (out.data_ptr(), out_split)
        return out, olens, None
