"""EBranchformerEncoder with the reference's constructor / state_dict surface, executed by the espnet_b200 CUDA kernels.

Reference: espnet2/asr/encoder/e_branchformer_encoder.py:55-563 (EBranchformerEncoderLayer, EBranchformerEncoder) and
espnet2/asr/layers/cgmlp.py:15-124 (ConvolutionalSpatialGatingUnit, ConvolutionalGatingMLP).  The attention branch is the Conformer's
rel-pos "latest" self-attention (band GEMM over a cached P_all, then the fused wgmma attention at d_k = 64); the cgMLP branch is
channel_proj1 with GELU in the GEMM epilogue, the CSGU kernel (LayerNorm + depthwise conv + gating, csrc/encoder_ops.cu) and
channel_proj2; the merge module is one depthwise-conv kernel over the concatenated branches followed by merge_proj.

Both branches write plain fp32 into one [M, 2D] buffer: the attention output (linear_out) into columns [0, D), channel_proj2 into
columns [D, 2D) -- the torch.cat of the reference.  The torch.nn layers are parameter containers only (reference checkpoints load by
name); forward never calls them.
"""
import math
from typing import List, Optional, Tuple

import torch

from . import ops
from .encoder import LN_EPS, _Conv2dSubsampling, _FFN, _PosBias, rel_pos_table
from .errors import TooShortUttError
from .lib import call, ptr
from .ops import ACT_GELU, ACT_RELU, ACT_SWISH, _count, gemm, layernorm, linear, new_split, split_from

_FFN_ACTS = {"swish": ACT_SWISH, "relu": ACT_RELU}   # get_activation (nets_utils.py:571-584) choices this path computes


class _CSGU(torch.nn.Module):
    def __init__(self, size, kernel_size):
        super().__init__()
        n = size // 2
        self.norm = torch.nn.LayerNorm(n, eps=LN_EPS)
        self.conv = torch.nn.Conv1d(n, n, kernel_size, 1, (kernel_size - 1) // 2, groups=n)


class _CgMLP(torch.nn.Module):
    def __init__(self, size, units, kernel_size):
        super().__init__()
        self.channel_proj1 = torch.nn.Sequential(torch.nn.Linear(size, units), torch.nn.GELU())
        self.csgu = _CSGU(units, kernel_size)
        self.channel_proj2 = torch.nn.Linear(units // 2, size)


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


class EBranchformerEncoder(torch.nn.Module):
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
        super().__init__()
        unsupported = []
        if input_layer != "conv2d": unsupported.append(f"input_layer={input_layer}")
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
        self._output_size, self.heads, self.num_blocks, self.idim = output_size, attention_heads, num_blocks, input_size
        self.cgmlp_units, self.cgmlp_kernel, self.merge_kernel = cgmlp_linear_units, cgmlp_conv_kernel, merge_conv_kernel
        self.ffn_units, self.use_ffn, self.macaron = linear_units, use_ffn, use_ffn and macaron_ffn
        self.ffn_act = _FFN_ACTS.get(ffn_activation_type, ACT_SWISH)
        self.ff_scale = 0.5 if self.macaron else 1.0
        self.embed = _Conv2dSubsampling(input_size, output_size)
        self.encoders = torch.nn.ModuleList(
            _Layer(output_size, attention_heads, cgmlp_linear_units, cgmlp_conv_kernel, linear_units, use_ffn, macaron_ffn, merge_conv_kernel)
            for _ in range(num_blocks))
        self.after_norm = torch.nn.LayerNorm(output_size, eps=LN_EPS)
        self._packed, self._ws, self._pos_cache = None, {}, {}
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
        D = C = self._output_size
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        e = self.embed
        F1 = (self.idim - 3) // 2 + 1
        F2 = (F1 - 3) // 2 + 1
        pk = dict(F1=F1, F2=F2, c1_w=f32(e.conv[0].weight).view(C, 9), c1_b=f32(e.conv[0].bias),
                  # conv2 weight [co][ci][kt][kf] -> [co][(kt*3+kf)*C + ci]
                  c2_w=split_from(f32(e.conv[2].weight).permute(0, 2, 3, 1).reshape(C, 9 * C)), c2_b=f32(e.conv[2].bias),
                  # embed.out columns are c*F2+f (subsampling.py:450-451) -> f*C+c to match the [B][F2][T][C] conv2 output
                  out_w=split_from(f32(e.out.weight).view(D, C, F2).permute(0, 2, 1).reshape(D, F2 * C)), out_b=f32(e.out.bias))
        ln = lambda m: (f32(m.weight), f32(m.bias))  # noqa: E731
        ffn = lambda m: (split_from(f32(m.w_1.weight)), f32(m.w_1.bias), split_from(f32(m.w_2.weight)), f32(m.w_2.bias))  # noqa: E731
        layers = []
        for lyr in self.encoders:
            a, cg = lyr.attn, lyr.cgmlp
            d = dict(norm_mha=ln(lyr.norm_mha), norm_mlp=ln(lyr.norm_mlp), norm_final=ln(lyr.norm_final))
            if self.use_ffn:
                d["norm_ff"], d["ffn"] = ln(lyr.norm_ff), ffn(lyr.feed_forward)
            if self.macaron:
                d["norm_ff_macaron"], d["ffn_macaron"] = ln(lyr.norm_ff_macaron), ffn(lyr.feed_forward_macaron)
            d["qkv_w"] = split_from(torch.cat([f32(a.linear_q.weight), f32(a.linear_k.weight), f32(a.linear_v.weight)], 0))
            d["qkv_b"] = torch.cat([f32(a.linear_q.bias), f32(a.linear_k.bias), f32(a.linear_v.bias)], 0)
            d["out_w"], d["out_b"] = split_from(f32(a.linear_out.weight)), f32(a.linear_out.bias)
            d["pos_u"], d["pos_v"] = f32(a.pos_bias_u).view(-1), f32(a.pos_bias_v).view(-1)
            d["p1_w"], d["p1_b"] = split_from(f32(cg.channel_proj1[0].weight)), f32(cg.channel_proj1[0].bias)
            d["csgu_ln"] = ln(cg.csgu.norm)
            d["csgu_w"], d["csgu_b"] = f32(cg.csgu.conv.weight).view(self.cgmlp_units // 2, -1), f32(cg.csgu.conv.bias)
            d["p2_w"], d["p2_b"] = split_from(f32(cg.channel_proj2.weight)), f32(cg.channel_proj2.bias)
            d["mg_w"], d["mg_b"] = f32(lyr.depthwise_conv_fusion.weight).view(2 * D, -1), f32(lyr.depthwise_conv_fusion.bias)
            d["mp_w"], d["mp_b"] = split_from(f32(lyr.merge_proj.weight)), f32(lyr.merge_proj.bias)
            layers.append(d)
        pk["layers"] = layers
        pk["pos_w_all"] = split_from(torch.cat([f32(l.attn.linear_pos.weight) for l in self.encoders], 0))  # [L*D][D]
        pk["after_norm"] = ln(self.after_norm)
        self._packed = pk
        return pk

    def _buf(self, name, shape, zero=False):
        key = (name, tuple(shape))
        t = self._ws.get(key)
        if t is None:
            t = (torch.zeros if zero else torch.empty)(shape, dtype=torch.float32, device=self.after_norm.weight.device)
            for k in [k for k in self._ws if k[0] == name and k != key]:   # drop stale buffers of the same name with other shapes
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

    def _ffn(self, x, xn, hbuf, norm, weights):
        """x += ff_scale * w_2(act(w_1(LN(x))))  (e_branchformer_encoder.py:132-135,172-176)."""
        w1, b1, w2, b2 = weights
        layernorm(x, *norm, LN_EPS, out_split=xn)
        linear(xn, w1, hbuf, bias=b1, act=self.ffn_act, split_out=True)
        linear(hbuf, w2, x, bias=b2, residual=x, alpha=self.ff_scale)

    # ---------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """xs_pad (B, T_f, idim) float32 CUDA (normalised log-mel), ilens (B,) -> (B, T, D), olens, None.

        Ragged batches follow per-utterance (batch-1) semantics of the reference: every utterance sees only its own frames (own attention
        keys, own conv boundaries in the CSGU and the merge module); rows t >= olens[b] of the output are 0."""
        pk = self._packed or self._pack()
        dev = xs_pad.device
        xs_pad = xs_pad.contiguous().float()
        B, Tf, F = xs_pad.shape
        assert F == self.idim
        # check_short_utt (subsampling.py:43-44), e_branchformer_encoder.py:482-499: the reference decodes one utterance per call, so the
        # limit applies to every utterance of a ragged batch, not to the padded length
        min_len = int(torch.as_tensor(ilens).min()) if torch.as_tensor(ilens).numel() else Tf
        if Tf < 7 or min_len < 7:
            size = min(Tf, min_len)
            which = "" if Tf < 7 else f" (utterance {int(torch.as_tensor(ilens).argmin())} of the batch)"
            raise TooShortUttError(f"has {size} frames and is too short for subsampling (it needs more than 7 frames), "
                                   f"return empty results{which}", size, 7)
        D, H, L, U = self._output_size, self.heads, self.num_blocks, self.cgmlp_units
        C, dk, Uh = D, D // H, U // 2
        F1, F2 = pk["F1"], pk["F2"]
        T1 = (Tf - 3) // 2 + 1
        T = (T1 - 3) // 2 + 1
        T1h, F1h = (T1 + 1) // 2, (F1 + 1) // 2
        olens = torch.div(torch.div(ilens - 1, 2, rounding_mode="trunc") - 1, 2, rounding_mode="trunc")
        lens32 = olens.to(device=dev, dtype=torch.int32).contiguous()
        M = B * T
        Tp, Rp = (T + 31) // 32 * 32, (2 * T - 1 + 31) // 32 * 32   # 128-byte row pitches of the score matrices (see encoder.py)

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
        hbuf = self._buf("h", (2, M, self.ffn_units)) if self.use_ffn else None
        qkv = self._buf("qkv", (2, M, 3 * D))
        qu, qv = self._buf("qu", (2, M, D)), self._buf("qv", (2, M, D))
        vt = self._buf("vt", (2, B, H, dk, Tp))
        bd = self._buf("bd", (B, H, T, Rp))
        fused = ops.use_flash_attn(dk)      # one wgmma kernel for q k^T + rel_shift + softmax + p v (csrc/attention.cu); else materialised
        if not fused:
            ac = self._buf("ac", (B, H, T, Tp))
            probs = self._buf("probs", (2, B, H, T, Tp))
        ctx = self._buf("ctx", (2, M, D))
        g1 = self._buf("g1", (M, U))              # channel_proj1 + GELU, plain
        stats = self._buf("stats", (M, 2))        # CSGU LayerNorm mean / rstd per row
        g2 = self._buf("g2", (2, M, Uh))          # CSGU output, split
        cat = self._buf("cat", (M, 2 * D))        # [x_att | x_cgmlp], plain
        mg = self._buf("mg", (2, M, 2 * D))       # cat + dwconv(cat), split
        for li, w in enumerate(pk["layers"]):
            if self.macaron:
                self._ffn(x, xn, hbuf, w["norm_ff_macaron"], w["ffn_macaron"])
            # branch 1: rel-pos MHSA (e_branchformer_encoder.py:141-152, attention.py:416-459) -> cat[:, :D]
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
            gemm(M, D, D, ctx, M * D, D, w["out_w"], D * D, D, cat, 2 * D, bias=w["out_b"])
            # branch 2: cgMLP (e_branchformer_encoder.py:154-163, cgmlp.py:110-124) -> cat[:, D:]
            layernorm(x, *w["norm_mlp"], LN_EPS, out_split=xn)
            linear(xn, w["p1_w"], g1, bias=w["p1_b"], act=ACT_GELU)
            call("espb_csgu_f32", ptr(g1), B, T, U, ptr(lens32), ptr(w["csgu_ln"][0]), ptr(w["csgu_ln"][1]), LN_EPS, ptr(w["csgu_w"]),
                 ptr(w["csgu_b"]), self.cgmlp_kernel, ptr(stats), ptr(g2), M * Uh)
            _count(2)
            gemm(M, D, Uh, g2, M * Uh, Uh, w["p2_w"], D * Uh, Uh, cat, 2 * D, bias=w["p2_b"], c_off=D)
            # merge: x += merge_proj(cat + dwconv(cat))  (e_branchformer_encoder.py:165-170)
            call("espb_merge_dwconv_f32", ptr(cat), B, T, 2 * D, ptr(lens32), ptr(w["mg_w"]), ptr(w["mg_b"]), self.merge_kernel, ptr(mg), M * 2 * D)
            _count()
            linear(mg, w["mp_w"], x, bias=w["mp_b"], residual=x)
            if self.use_ffn:
                self._ffn(x, xn, hbuf, w["norm_ff"], w["ffn"])
            layernorm(x, *w["norm_final"], LN_EPS, out_plain=x)
            if self.trace is not None:
                self.trace.append(x.view(B, T, D).clone())
        out = torch.empty(B, T, D, dtype=torch.float32, device=dev)
        out_split = self._buf("enc_split", (2, M, D))
        layernorm(x, *pk["after_norm"], LN_EPS, out_plain=out, out_split=out_split)
        call("espb_zero_pad_rows_f32", ptr(out), B, T, D, ptr(lens32), 0, 1)
        call("espb_zero_pad_rows_f32", ptr(out_split), B, T, D, ptr(lens32), M * D, 2)
        _count(2)
        self.last_split_out = (out.data_ptr(), out_split)
        return out, olens, None
