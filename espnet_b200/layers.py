"""Host code the CUDA-path modules share: the parameter containers (the reference's attribute names, created in the reference's order so
that a seeded default init gives the same weights), the sinusoid tables, ``PackedModule`` -- the packed weights and workspace of every
encoder, decoder, LM and CTC head, the packing of LayerNorm, attention and feed-forward weights and the feed-forward launches -- and
``EncoderBase``, the state every encoder has (``after_norm``) and the packing and launches of the blocks they have in common:
Conv2dSubsampling, the convolution module, rel-pos and plain self-attention.  Each encoder module keeps its constructor checks, its layer
container, the packing of its own weights and its per-layer sequence in ``forward``.

The torch.nn layers are parameter containers only (reference checkpoints load by name); forward never calls them.
"""
import math

import torch

from . import ops
from .errors import TooShortUttError
from .ops import ACT_GELU, ACT_RELU, _count, layernorm, linear, split_from

# Launches go through ops.call / ops.ptr / ops.gemm / ops.new_split, looked up at call time: the kernel emulation of the tests
# (tests/emu_backend.py) replaces them in ops and in each encoder module.

LN_EPS = 1e-12  # transformer/layer_norm.py:22


class _MHA(torch.nn.Module):
    def __init__(self, n_feat):
        super().__init__()
        self.linear_q = torch.nn.Linear(n_feat, n_feat)
        self.linear_k = torch.nn.Linear(n_feat, n_feat)
        self.linear_v = torch.nn.Linear(n_feat, n_feat)
        self.linear_out = torch.nn.Linear(n_feat, n_feat)


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


class _CSGU(torch.nn.Module):
    def __init__(self, size, kernel_size):
        super().__init__()
        n = size // 2
        self.norm = torch.nn.LayerNorm(n, eps=LN_EPS)
        self.conv = torch.nn.Conv1d(n, n, kernel_size, 1, (kernel_size - 1) // 2, groups=n)


class _CgMLP(torch.nn.Module):
    """ConvolutionalGatingMLP (cgmlp.py:84-124) with the identity gate and no linear after the conv."""

    def __init__(self, size, units, kernel_size):
        super().__init__()
        self.channel_proj1 = torch.nn.Sequential(torch.nn.Linear(size, units), torch.nn.GELU())
        self.csgu = _CSGU(units, kernel_size)
        self.channel_proj2 = torch.nn.Linear(units // 2, size)


# input_layer -> (kernel, stride) of the convs after the first Conv2d(1, odim, 3, 2) (subsampling.py:386-860), and check_short_utt's limit
# (subsampling.py:31-48): the fewest input frames that leave one output frame.
SUBSAMPLING = {"conv2d": ((3, 2),), "conv2d2": ((3, 1),), "conv2d6": ((5, 3),), "conv2d8": ((3, 2), (3, 2))}
MIN_FRAMES = {"conv2d": 7, "conv2d2": 7, "conv2d6": 11, "conv2d8": 15}
_A_MODE = {(3, 2): 1, (3, 1): 2, (5, 3): 3}   # (kernel, stride) -> EspbGemmDesc.a_mode of the implicit-GEMM conv (gemm.h: conv_geom)


class _Conv2dSubsampling(torch.nn.Module):
    """Conv2dSubsampling{,2,6,8} and Conv2dSubsamplingWOPosEnc: conv.0 / conv.2 (/ conv.4) and out, sized by the input layer (the
    positional encoding has no parameters)."""

    def __init__(self, idim, odim, input_layer="conv2d"):
        super().__init__()
        convs = [torch.nn.Conv2d(1, odim, 3, 2), torch.nn.ReLU()]
        for k, s in SUBSAMPLING[input_layer]:
            convs += [torch.nn.Conv2d(odim, odim, k, s), torch.nn.ReLU()]
        self.conv = torch.nn.Sequential(*convs)
        self.out = torch.nn.Linear(odim * subsampled_len(idim, input_layer)[-1], odim)


def _sinusoid_table(pos, d):
    """Row k = sin / cos of pos[k] * 10000^(-2i/d) in the even / odd columns (embedding.py:62-83)."""
    pos = pos.unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe = torch.zeros(pos.shape[0], d)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


def abs_pos_table(length, d):
    """PositionalEncoding.extend_pe (embedding.py:62-83): row t = sinusoid of position t."""
    return _sinusoid_table(torch.arange(0, length, dtype=torch.float32), d)


def rel_pos_table(T, d):
    """(2T-1, d) slice RelPositionalEncoding.forward returns: row k = sinusoid of relative position T-1-k
    (embedding.py:286-334).  Built once per length on the host, like the reference's ``pe`` buffer."""
    return _sinusoid_table(torch.arange(T - 1, -T, -1, dtype=torch.float32), d)


def subsampled_len(n, input_layer="conv2d"):
    """Lengths after each conv of the input layer's subsampling (after conv1, after conv2[, after conv3]); n an int or an integer tensor."""
    out = [(n - 3) // 2 + 1]
    for k, s in SUBSAMPLING[input_layer]:
        out.append((out[-1] - k) // s + 1)
    return tuple(out)


def _pitch(n):
    """Row pitch of the score / probability matrices: a multiple of 32 floats, so that every 128-byte store segment of the GEMM epilogues
    is a whole cache line (partial-sector writes cost a DRAM read-modify-write)."""
    return (n + 31) // 32 * 32


class PackedModule(torch.nn.Module):
    """A module whose forward runs the kernels on device-side copies of its weights (``_packed``, built by the subclass's ``_pack`` and
    dropped when a state_dict loads) and on a workspace of named buffers kept across calls (``_buf``)."""

    ws_tag = 0          # workspace set in use: the search runs independent utterance groups on separate streams, each with its own buffers
    zero_bufs = False   # True: every workspace buffer is zero-filled when (re)created, not only those asked for with zero=True

    def __init__(self):
        super().__init__()
        self._packed, self._ws = None, {}
        self.buf_version = 0   # bumped on every allocation: captured CUDA graphs hold the buffers' pointers

    def _load_from_state_dict(self, *args, **kwargs):
        self._packed = None
        return super()._load_from_state_dict(*args, **kwargs)

    @property
    def _device(self):
        return next(self.parameters()).device

    def _buf(self, name, shape, zero=False, dtype=torch.float32):
        """Workspace tensor kept across calls; a new shape or dtype replaces the buffer of that name (freed before the allocation)."""
        name = (self.ws_tag, name)
        key = (name, tuple(shape), dtype)
        t = self._ws.get(key)
        if t is None:
            for k in [k for k in self._ws if k[0] == name]:
                del self._ws[k]
            t = (torch.zeros if zero or self.zero_bufs else torch.empty)(shape, dtype=dtype, device=self._device)
            self._ws[key] = t
            self.buf_version += 1
        return t

    # ---------------------------------------------------------------- weights -> device-side packed/split form
    def _f32(self, t):
        return t.detach().to(device=self._device, dtype=torch.float32).contiguous()

    def _pack_ln(self, m):
        return self._f32(m.weight), self._f32(m.bias)

    def _pack_ffn(self, m):
        f32 = self._f32
        return split_from(f32(m.w_1.weight)), f32(m.w_1.bias), split_from(f32(m.w_2.weight)), f32(m.w_2.bias)

    def _pack_mha(self, a):
        """q / k / v projections fused into one [3D][D] GEMM, linear_out, and the rel-pos biases of a _PosBias."""
        f32 = self._f32
        d = dict(qkv_w=split_from(torch.cat([f32(a.linear_q.weight), f32(a.linear_k.weight), f32(a.linear_v.weight)], 0)),
                 qkv_b=torch.cat([f32(a.linear_q.bias), f32(a.linear_k.bias), f32(a.linear_v.bias)], 0),
                 out_w=split_from(f32(a.linear_out.weight)), out_b=f32(a.linear_out.bias))
        if isinstance(a, _PosBias):
            d["pos_u"], d["pos_v"] = f32(a.pos_bias_u).view(-1), f32(a.pos_bias_v).view(-1)
        return d

    # ---------------------------------------------------------------- launches
    def _ffn(self, x, xn, norm, weights, act, alpha=1.0):
        """x += alpha * w_2(act(w_1(LN(x))))  (PositionwiseFeedForward behind its pre-LayerNorm)."""
        w1, b1, w2, b2 = weights
        h = self._buf("h", (2, x.shape[0], w1.shape[1]))
        layernorm(x, *norm, LN_EPS, out_split=xn)
        linear(xn, w1, h, bias=b1, act=act, split_out=True)
        linear(h, w2, x, bias=b2, residual=x, alpha=alpha)


class EncoderBase(PackedModule):
    """``embed`` (Conv2dSubsampling), ``encoders`` (the layers, built from ``layers``) and ``after_norm``, created in this order as in the
    reference.  Subclasses set ``heads`` and ``num_blocks`` (and ``kernel`` with the convolution module) and define ``_pack`` and
    ``forward``."""

    trace = None            # set to a list to collect per-stage outputs (tests)
    last_split_out = None   # split copy of the last output (feeds the CTC head / decoder memory GEMMs)

    def __init__(self, input_size, output_size, layers, input_layer="conv2d"):
        super().__init__()
        self._output_size, self.idim, self.input_layer = output_size, input_size, input_layer
        self.embed = _Conv2dSubsampling(input_size, output_size, input_layer)
        self.encoders = torch.nn.ModuleList(layers)
        self.after_norm = torch.nn.LayerNorm(output_size, eps=LN_EPS)
        self._pos_cache = {}   # rel-pos encoders: _pos per length

    def output_size(self) -> int:
        return self._output_size

    def _init_interctc(self, interctc_layer_idx, interctc_use_conditioning, num_blocks):
        """Intermediate CTC (conformer_encoder.py:317-321): after each listed block (1-based) the encoder returns after_norm(x) and, with
        conditioning, feeds the CTC posteriors back into x through ``conditioning_layer``, which ESPnetASRModel creates."""
        self.interctc_layer_idx = list(interctc_layer_idx)
        if len(self.interctc_layer_idx) > 0:
            assert 0 < min(self.interctc_layer_idx) and max(self.interctc_layer_idx) < num_blocks
        self.interctc_use_conditioning = interctc_use_conditioning
        self.conditioning_layer = None

    def _check_interctc(self, ctc):
        if self.interctc_layer_idx and self.interctc_use_conditioning:
            if ctc is None:
                raise ValueError(f"{type(self).__name__} with interctc_use_conditioning needs the CTC head: call it as encoder(xs_pad, ilens, "
                                 "ctc=model.ctc)")
            if self.conditioning_layer is None:
                raise ValueError(f"{type(self).__name__} with interctc_use_conditioning has no conditioning_layer: ESPnetASRModel creates it "
                                 "(Linear(vocab_size, output_size))")
            if self.conditioning_layer.in_features != ctc.odim:
                raise ValueError(f"conditioning_layer takes {self.conditioning_layer.in_features} posteriors, the CTC head has {ctc.odim}")
            if self._packed is not None and "cond_w" not in self._packed:   # conditioning_layer set after the weights were packed
                self._packed = None

    def _pack_pos(self, attns):
        """linear_pos of every attention layer stacked [L*D][D], L = the number of attention layers (layer ordinal a at rows a*D..): one GEMM
        per length projects the rel-pos table for all of them (_pos)."""
        return split_from(torch.cat([self._f32(a.linear_pos.weight) for a in attns], 0))

    def _pack_cgmlp(self, cg):
        """channel_proj1, the CSGU's LayerNorm and depthwise conv, channel_proj2 of a _CgMLP."""
        f32 = self._f32
        return dict(p1_w=split_from(f32(cg.channel_proj1[0].weight)), p1_b=f32(cg.channel_proj1[0].bias), csgu_ln=self._pack_ln(cg.csgu.norm),
                    csgu_w=f32(cg.csgu.conv.weight).view(cg.csgu.conv.weight.shape[0], -1), csgu_b=f32(cg.csgu.conv.bias),
                    p2_w=split_from(f32(cg.channel_proj2.weight)), p2_b=f32(cg.channel_proj2.bias))

    def _pack_conv(self, cm):
        f32, D = self._f32, self._output_size
        d = dict(pw1_w=split_from(f32(cm.pointwise_conv1.weight).view(2 * D, D)), pw1_b=f32(cm.pointwise_conv1.bias),
                 dw_w=f32(cm.depthwise_conv.weight).view(D, -1), dw_b=f32(cm.depthwise_conv.bias))
        # BatchNorm1d eval: y = x*alpha + beta with alpha = weight/sqrt(var+eps) (what ATen's CPU kernel computes)
        inv = 1.0 / torch.sqrt(f32(cm.norm.running_var) + cm.norm.eps)
        alpha = inv * f32(cm.norm.weight)
        d["bn_a"], d["bn_b"] = alpha.contiguous(), (f32(cm.norm.bias) - f32(cm.norm.running_mean) * alpha).contiguous()
        d["pw2_w"], d["pw2_b"] = split_from(f32(cm.pointwise_conv2.weight).view(D, D)), f32(cm.pointwise_conv2.bias)
        return d

    def _pack_io(self):
        """Conv2dSubsampling in the layouts of the conv1 kernel and the implicit-GEMM convs, after_norm, and conditioning_layer if set."""
        f32, e = self._f32, self.embed
        D = C = self._output_size
        Fs = subsampled_len(self.idim, self.input_layer)
        convs = []
        for i, (k, _) in enumerate(SUBSAMPLING[self.input_layer]):
            # weight [co][ci][kt][kf] -> [co][(kt*k+kf)*C + ci]
            cv = e.conv[2 * i + 2]
            convs.append((split_from(f32(cv.weight).permute(0, 2, 3, 1).reshape(C, k * k * C)), f32(cv.bias)))
        return dict(F=Fs, c1_w=f32(e.conv[0].weight).view(C, 9), c1_b=f32(e.conv[0].bias), convs=convs,
                    # embed.out columns are c*F+f (subsampling.py:450-451) -> f*C+c to match the [B][F][T][C] output of the last conv
                    out_w=split_from(f32(e.out.weight).view(D, C, Fs[-1]).permute(0, 2, 1).reshape(D, Fs[-1] * C)), out_b=f32(e.out.bias),
                    after_norm=self._pack_ln(self.after_norm), **self._pack_cond())

    def _pack_cond(self):
        """conditioning_layer [D][V] as the B operand of a GEMM with K = _pitch(V): zero columns V.. meet the zero columns of the posteriors."""
        cl = getattr(self, "conditioning_layer", None)
        if cl is None:
            return {}
        w = self._f32(cl.weight)
        wp = torch.zeros(w.shape[0], _pitch(w.shape[1]), dtype=torch.float32, device=w.device)
        wp[:, : w.shape[1]] = w
        return dict(cond_w=split_from(wp), cond_b=self._f32(cl.bias))

    # ---------------------------------------------------------------- launches
    def _lengths(self, xs_pad, ilens):
        """check_short_utt (subsampling.py:31-48) and the subsampled lengths -> (xs_pad fp32 contiguous, T, olens, lens32 on the device).

        The reference decodes one utterance per call, so the limit applies to every utterance of a ragged batch, not to the padded length
        (an utterance below the limit would get olens 0)."""
        xs_pad = xs_pad.contiguous().float()
        B, Tf, F = xs_pad.shape
        assert F == self.idim
        lim = MIN_FRAMES[self.input_layer]
        min_len = int(torch.as_tensor(ilens).min()) if torch.as_tensor(ilens).numel() else Tf
        if Tf < lim or min_len < lim:
            size = min(Tf, min_len)
            which = "" if Tf < lim else f" (utterance {int(torch.as_tensor(ilens).argmin())} of the batch)"
            raise TooShortUttError(f"has {size} frames and is too short for subsampling (it needs more than {lim} frames), "
                                   f"return empty results{which}", size, lim)
        olens = subsampled_len(torch.as_tensor(ilens), self.input_layer)[-1]
        return xs_pad, subsampled_len(Tf, self.input_layer)[-1], olens, olens.to(device=xs_pad.device, dtype=torch.int32).contiguous()

    def _subsample(self, xs, x, alpha, pe=None):
        """Conv2dSubsampling{,2,6,8} (subsampling.py:432-474, 625-649, 730-754, 838-862) of xs (B, T_f, idim) into x [B*T][D]:
        x = alpha * out(conv(xs)) [+ pe[t]], the positional table entering as a batch-broadcast residual of the embed.out GEMM.

        conv1 writes its output split into the phases of the next conv's stride; each following conv is an implicit GEMM over such a
        phase-split input (one output frequency per batch x slice), and its split [B][F][T][C] output is re-laid into phases when another
        strided conv follows (conv2d8)."""
        pk = self._packed
        B, Tf, F = xs.shape
        D = C = self._output_size
        geo = SUBSAMPLING[self.input_layer]
        Fs, Ts = pk["F"], subsampled_len(Tf, self.input_layer)
        s = geo[0][1]
        Th, Fh = -(-Ts[0] // s), -(-Fs[0] // s)
        a = self._buf("c1", (B, 2 * s * s, Fh, Th, C), zero=True)
        if s == 2:   # the parity split (conv2d, conv2d8): the s = 2 entry point of the same kernel
            ops.call("espb_conv1_relu_f32", ops.ptr(xs), B, Tf, F, ops.ptr(pk["c1_w"]), ops.ptr(pk["c1_b"]), C, ops.ptr(a), Ts[0], Fs[0], Th, Fh)
        else:
            ops.call("espb_conv1_relu_phase_f32", ops.ptr(xs), B, Tf, F, ops.ptr(pk["c1_w"]), ops.ptr(pk["c1_b"]), C, ops.ptr(a), Ts[0], Fs[0],
                     s, Th, Fh)
        _count()
        for i, ((k, s), (w, b)) in enumerate(zip(geo, pk["convs"])):
            To, Fo = Ts[i + 1], Fs[i + 1]
            c = self._buf(f"c{i + 2}", (2, B, Fo, To, C))
            ops.gemm(To, C, k * k * C, a, 0, 0, w, C * k * k * C, k * k * C, c, C, c_plane=B * Fo * To * C, split_out=True, bias=b,
                     act=ACT_RELU, nbx=Fo, nby=B, sc=(To * C, Fo * To * C), a_mode=_A_MODE[(k, s)], conv=(Th, Fh, C))
            if i + 1 < len(geo):
                s = geo[i + 1][1]
                Th, Fh = -(-To // s), -(-Fo // s)
                a = self._buf(f"c{i + 2}p", (B, 2 * s * s, Fh, Th, C), zero=True)
                ops.call("espb_phase_split_f32", ops.ptr(c), B * Fo * To * C, B, Fo, To, C, s, Th, Fh, ops.ptr(a))
                _count()
        T, Fl = Ts[-1], Fs[-1]
        ops.gemm(T, D, Fl * C, c, B * Fl * T * C, C, pk["out_w"], D * Fl * C, Fl * C, x, D, bias=pk["out_b"], alpha=alpha, R=pe,
                 ldr=0 if pe is None else D, nbx=1, nby=B, sa=(T * C, Fl * T * C), sc=(0, T * D), kob=C // 32)

    def _conv_module(self, x, xn, norm, w, nseq, S, lens):
        """x += ConvolutionModule(LN(x))  (convolution.py:56-79) over nseq sequences of S rows; sequence b sees zeros outside rows
        0..lens[b]-1.  GLU, depthwise conv, BatchNorm and swish run as one kernel between the two pointwise GEMMs."""
        D, M = self._output_size, nseq * S
        y, cv = self._buf("y", (M, 2 * D)), self._buf("cv", (2, M, D))
        layernorm(x, *norm, LN_EPS, out_split=xn)
        linear(xn, w["pw1_w"], y, bias=w["pw1_b"])
        ops.call("espb_glu_dwconv_bn_swish_f32", ops.ptr(y), nseq, S, D, ops.ptr(lens), ops.ptr(w["dw_w"]), ops.ptr(w["dw_b"]), self.kernel,
                 ops.ptr(w["bn_a"]), ops.ptr(w["bn_b"]), ops.ptr(cv), M * D)
        _count()
        linear(cv, w["pw2_w"], x, bias=w["pw2_b"], residual=x)

    def _cgmlp(self, x, xn, w, B, T, lens32, out, ldc, c_off=0, split_out=False, residual=None):
        """ConvolutionalGatingMLP(norm_mlp(x)) (cgmlp.py:110-124) of the M = B*T rows of x into out[:, c_off:c_off + D] (row stride ldc; a
        split out has planes of M*ldc), plus residual when given: norm_mlp, channel_proj1 with GELU in the epilogue, the CSGU kernel
        (LayerNorm + depthwise conv + gating, each utterance seeing zeros outside its own rows), channel_proj2."""
        D, U, K = self._output_size, self.cgmlp_units, self.cgmlp_kernel
        M, Uh = B * T, U // 2
        g1 = self._buf("g1", (M, U))              # channel_proj1 + GELU, plain
        stats = self._buf("stats", (M, 2))        # CSGU LayerNorm mean / rstd per row
        g2 = self._buf("g2", (2, M, Uh))          # CSGU output, split
        layernorm(x, *w["norm_mlp"], LN_EPS, out_split=xn)
        linear(xn, w["p1_w"], g1, bias=w["p1_b"], act=ACT_GELU)
        ops.call("espb_csgu_f32", ops.ptr(g1), B, T, U, ops.ptr(lens32), ops.ptr(w["csgu_ln"][0]), ops.ptr(w["csgu_ln"][1]), LN_EPS,
                 ops.ptr(w["csgu_w"]), ops.ptr(w["csgu_b"]), K, ops.ptr(stats), ops.ptr(g2), M * Uh)
        _count(2)
        ops.gemm(M, D, Uh, g2, M * Uh, Uh, w["p2_w"], D * Uh, Uh, out, ldc, c_plane=M * ldc if split_out else 0, split_out=split_out,
                 bias=w["p2_b"], R=residual, ldr=D if residual is not None else 0, c_off=c_off)

    def _pos(self, T):
        """P_all split [2][2T-1][L*D] = linear_pos(pos_emb) for every attention layer (one GEMM per length, cached); L*D is the width of
        the packed pos_w_all."""
        if T not in self._pos_cache:
            if len(self._pos_cache) > 8:
                self._pos_cache.clear()
            D, LD = self._output_size, self._packed["pos_w_all"].shape[1]
            pe = split_from(rel_pos_table(T, D).to(self._device))
            out = ops.new_split(2 * T - 1, LD, device=pe.device)
            linear(pe, self._packed["pos_w_all"], out, split_out=True)
            self._pos_cache[T] = out
        return self._pos_cache[T]

    def _relpos_attn(self, qkv, w, li, p_all, ctx, B, T, lens32):
        """RelPositionMultiHeadedAttention (attention.py:416-459) of attention layer li (its ordinal among the layers with attention, which
        is the layer index in an encoder where every layer has one), from the fused q|k|v projection qkv (split [2][B*T][3D]) to ctx (split
        [2][B*T][D]); the output projection is the caller's.  p_all = _pos(T)."""
        D, H = self._output_size, self.heads
        dk, M, R = D // H, B * T, 2 * T - 1
        L = p_all.shape[2] // D
        Tp, Rp = _pitch(T), _pitch(R)
        qu, qv = self._buf("qu", (2, M, D)), self._buf("qv", (2, M, D))
        vt = self._buf("vt", (2, B, H, dk, Tp))
        bd = self._buf("bd", (B, H, T, Rp))
        ops.call("espb_qu_qv_f32", ops.ptr(qkv), M * 3 * D, M, D, ops.ptr(w["pos_u"]), ops.ptr(w["pos_v"]), ops.ptr(qu), ops.ptr(qv), M * D)
        ops.call("espb_v_transpose_f32", ops.ptr(qkv), M * 3 * D, B, T, D, H, ops.ptr(lens32), ops.ptr(vt), B * H * dk * Tp, Tp)
        _count(2)
        ops.gemm(T, R, dk, qv, M * D, D, p_all, R * L * D, L * D, bd, Rp, nbx=H, nby=B, sa=(dk, T * D), sb=(dk, 0),
                 sc=(T * Rp, H * T * Rp), b_off=li * D, band_t=T)   # rel_shift only ever reads bd[i][T-1-i .. 2T-2-i]
        if ops.use_flash_attn(dk):      # one wgmma kernel for q k^T + rel_shift + softmax + p v (csrc/attention.cu); else materialised
            ops.flash_attn(qu, 0, D, qkv, D, 3 * D, vt, Tp, bd, Rp, lens32, B, H, T, dk, ctx)
        else:
            ac, probs = self._buf("ac", (B, H, T, Tp)), self._buf("probs", (2, B, H, T, Tp))
            ops.gemm(T, T, dk, qu, M * D, D, qkv, M * 3 * D, 3 * D, ac, Tp, nbx=H, nby=B, sa=(dk, T * D), sb=(dk, T * 3 * D),
                     sc=(T * Tp, H * T * Tp), b_off=D)
            ops.call("espb_relpos_softmax_f32", ops.ptr(ac), ops.ptr(bd), B, H, T, Tp, Rp, ops.ptr(lens32), math.sqrt(dk), ops.ptr(probs),
                     B * H * T * Tp)
            _count()
            ops.gemm(T, dk, T, probs, B * H * T * Tp, Tp, vt, B * H * dk * Tp, Tp, ctx, D, c_plane=M * D, split_out=True, nbx=H, nby=B,
                     sa=(T * Tp, H * T * Tp), sb=(dk * Tp, H * dk * Tp), sc=(dk, T * D))

    def _attn(self, qkv, ctx, nseq, S, lens, fused):
        """MultiHeadedAttention (attention.py:77-151) over nseq sequences of S rows, from the fused q|k|v projection qkv (split
        [2][nseq*S][3D]) to ctx (split [2][nseq*S][D]); sequence b attends its keys 0..lens[b]-1.  fused: one wgmma kernel for q k^T + masked
        softmax + p v (csrc/attention.cu); else scores and probabilities are materialised.  The output projection is the caller's."""
        D, H = self._output_size, self.heads
        dk, M, Sp = D // H, nseq * S, _pitch(S)
        vt = self._buf("vt", (2, nseq, H, dk, Sp))
        ops.call("espb_v_transpose_f32", ops.ptr(qkv), M * 3 * D, nseq, S, D, H, ops.ptr(lens), ops.ptr(vt), nseq * H * dk * Sp, Sp)
        _count()
        if fused:
            ops.flash_attn(qkv, 0, 3 * D, qkv, D, 3 * D, vt, Sp, None, 0, lens, nseq, H, S, dk, ctx)
        else:
            sc, probs = self._buf("sc", (nseq, H, S, Sp)), self._buf("probs", (2, nseq, H, S, Sp))
            ops.gemm(S, S, dk, qkv, M * 3 * D, 3 * D, qkv, M * 3 * D, 3 * D, sc, Sp, nbx=H, nby=nseq, sa=(dk, S * 3 * D), sb=(dk, S * 3 * D),
                     sc=(S * Sp, H * S * Sp), b_off=D)
            ops.call("espb_masked_softmax_f32", ops.ptr(sc), nseq, H, S, Sp, ops.ptr(lens), math.sqrt(dk), ops.ptr(probs), nseq * H * S * Sp)
            _count()
            ops.gemm(S, dk, S, probs, nseq * H * S * Sp, Sp, vt, nseq * H * dk * Sp, Sp, ctx, D, c_plane=M * D, split_out=True, nbx=H, nby=nseq,
                     sa=(S * Sp, H * S * Sp), sb=(dk * Sp, H * dk * Sp), sc=(dk, S * D))

    def _interctc(self, x, B, T, ctc):
        """After a block listed in interctc_layer_idx (conformer_encoder.py:391-414, transformer_encoder.py:279-291): returns the intermediate
        output after_norm(x) as a new (B, T, D) tensor and, with conditioning, adds conditioning_layer(softmax(ctc_lo(after_norm(x)))) to x.
        The posteriors go straight into the split A operand of the conditioning GEMM, zero-padded to a K that is a multiple of 32.  Every
        step is row-wise, so padding rows of a ragged batch only reach padding rows."""
        D, M = self._output_size, B * T
        h = torch.empty(B, T, D, dtype=torch.float32, device=x.device)
        if not self.interctc_use_conditioning:
            layernorm(x, *self._packed["after_norm"], LN_EPS, out_plain=h)
            return h
        V = ctc.odim
        hs = self._buf("ic_split", (2, M, D))
        logits, probs = self._buf("ic_logits", (M, V)), self._buf("ic_probs", (2, M, _pitch(V)))
        layernorm(x, *self._packed["after_norm"], LN_EPS, out_plain=h, out_split=hs)
        ctc.logits(h, hs, out=logits)
        ops.softmax_rows_split(logits, probs)
        linear(probs, self._packed["cond_w"], x, bias=self._packed["cond_b"], residual=x)
        return h

    def _output(self, x, B, T):
        """after_norm into a new (B, T, D) tensor and its split copy (last_split_out) -> (out, out_split)."""
        D = self._output_size
        out = torch.empty(B, T, D, dtype=torch.float32, device=x.device)
        out_split = self._buf("enc_split", (2, B * T, D))
        layernorm(x, *self._packed["after_norm"], LN_EPS, out_plain=out, out_split=out_split)
        self.last_split_out = (out.data_ptr(), out_split)
        return out, out_split
