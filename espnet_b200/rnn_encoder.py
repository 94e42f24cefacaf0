"""VGGRNNEncoder and RNNEncoder (the classic ESPnet RNN encoders) with the reference's constructor / state_dict surface, executed by the
espnet_b200 CUDA kernels.

Reference: espnet2/asr/encoder/vgg_rnn_encoder.py, espnet2/asr/encoder/rnn_encoder.py and the legacy modules they compose
(legacy/nets/pytorch_backend/rnn/encoders.py: VGG2L, RNNP, RNN).  LSTM cells only (``rnn_type: gru`` is refused), uni- or bidirectional,
with or without per-layer projections; RNNEncoder also with frame subsampling between layers.

Every utterance of a ragged batch gets what decoding it alone gives (the reference runs the LSTMs through pack_padded_sequence): the VGG
convs see zeros past the utterance's own length, the pools and their ``ceil(len / 2)`` lengths are per utterance, and the backward
direction of each utterance starts at its own last frame.

Layout of the work:
  * VGG2L: conv1_1 (one input channel) is a direct kernel; conv1_2, conv2_1 and conv2_2 are implicit GEMMs (EspbGemmDesc a_mode 2, a
    stride-1 3x3 window) over a zero-bordered split input, so the padding costs no branch; the pools (and the re-bordering of conv2_1's
    output) are one kernel each, the last one writing the (channel, freq)-flattened rows the first LSTM input GEMM reads.
  * each LSTM layer: one GEMM for the input-to-gate products of every frame and both directions, then per time step one GEMM
    h_{t-1} W_hh^T for both directions (directions as GEMM batch) and one cell kernel: 2 launches per step.
  * projections: one GEMM each, then a kernel for tanh, the zeroed padding rows and the split copy the next GEMM reads.
The torch.nn layers are parameter containers only (reference checkpoints load by name); forward never calls them.
"""
import math
from typing import Optional, Sequence, Tuple

import torch

from . import ops
from .layers import PackedModule
from .ops import ACT_RELU, _count, split_from


def _pad4(k):
    return (k + 3) & ~3


def vgg2l_odim(idim, in_channel=1):
    """get_vgg2l_odim (legacy/nets/e2e_asr_common.py): 128 channels x the frequency extent after two ceil-mode pools."""
    idim = idim / in_channel
    idim = math.ceil(float(idim) / 2)
    idim = math.ceil(float(idim) / 2)
    return int(idim) * 128


class _LSTMParams(torch.nn.Module):
    """nn.LSTM's parameters under nn.LSTM's names (weight_ih_l{k}[_reverse], ...) without being an nn.LSTM (which re-flattens its weights
    through cuDNN on the GPU).  Created in nn.LSTM's order with its default init, so a seeded construction draws what nn.LSTM draws."""

    def __init__(self, idim, hidden, layers, bidirectional):
        super().__init__()
        ndir = 2 if bidirectional else 1
        for k in range(layers):
            isz = idim if k == 0 else hidden * ndir
            for sfx in ("", "_reverse")[:ndir]:
                self.register_parameter(f"weight_ih_l{k}{sfx}", torch.nn.Parameter(torch.empty(4 * hidden, isz)))
                self.register_parameter(f"weight_hh_l{k}{sfx}", torch.nn.Parameter(torch.empty(4 * hidden, hidden)))
                self.register_parameter(f"bias_ih_l{k}{sfx}", torch.nn.Parameter(torch.empty(4 * hidden)))
                self.register_parameter(f"bias_hh_l{k}{sfx}", torch.nn.Parameter(torch.empty(4 * hidden)))
        bound = 1.0 / math.sqrt(hidden)
        for p in self.parameters():
            torch.nn.init.uniform_(p, -bound, bound)


class _VGG2L(torch.nn.Module):
    def __init__(self, in_channel=1):
        super().__init__()
        self.conv1_1 = torch.nn.Conv2d(in_channel, 64, 3, stride=1, padding=1)
        self.conv1_2 = torch.nn.Conv2d(64, 64, 3, stride=1, padding=1)
        self.conv2_1 = torch.nn.Conv2d(64, 128, 3, stride=1, padding=1)
        self.conv2_2 = torch.nn.Conv2d(128, 128, 3, stride=1, padding=1)


class _RNNP(torch.nn.Module):
    """RNNP's parameters: per layer a 1-layer (B)LSTM ``birnn{i}`` / ``rnn{i}`` and its projection ``bt{i}``."""

    def __init__(self, idim, elayers, cdim, hdim, bidir):
        super().__init__()
        for i in range(elayers):
            setattr(self, f"{'birnn' if bidir else 'rnn'}{i}", _LSTMParams(idim if i == 0 else hdim, cdim, 1, bidir))
            setattr(self, f"bt{i}", torch.nn.Linear(2 * cdim if bidir else cdim, hdim))


class _RNN(torch.nn.Module):
    """RNN's parameters: one stacked (B)LSTM ``nbrnn`` and ``l_last``."""

    def __init__(self, idim, elayers, cdim, hdim, bidir):
        super().__init__()
        self.nbrnn = _LSTMParams(idim, cdim, elayers, bidir)
        self.l_last = torch.nn.Linear(2 * cdim if bidir else cdim, hdim)


class _RNNEncoderBase(PackedModule):
    trace = None            # set to a list to collect per-stage outputs (tests)
    last_split_out = None   # split copy of the last output (feeds the CTC head / decoder memory GEMMs)

    def _init_common(self, input_size, rnn_type, bidirectional, use_projection, num_layers, hidden_size, output_size):
        if rnn_type not in {"lstm", "gru"}:
            raise ValueError(f"Not supported rnn_type={rnn_type}")
        if rnn_type == "gru":
            raise NotImplementedError(f"espnet_b200.{type(self).__name__} implements rnn_type lstm (got gru)")
        self._output_size, self.idim = output_size, input_size
        self.rnn_type, self.bidirectional, self.use_projection = rnn_type, bidirectional, use_projection
        self.num_layers, self.hidden_size = num_layers, hidden_size
        self.ndir = 2 if bidirectional else 1

    def output_size(self) -> int:
        return self._output_size

    def _rnn_module(self):
        return self.enc[-1]

    # ---------------------------------------------------------------- packing
    def _pack_lstm(self, p, k, isz):
        """Layer k of an _LSTMParams: W_ih of both directions stacked [ndir*4H][pad4(isz)] with b_ih + b_hh, W_hh [ndir][4H][Hp]."""
        f32, dev, H = self._f32, self._device, self.hidden_size
        Hp, Kp = _pad4(H), _pad4(isz)
        sfx = ("", "_reverse")[:self.ndir]
        wih = torch.zeros(self.ndir * 4 * H, Kp, dtype=torch.float32, device=dev)
        whh = torch.zeros(self.ndir, 4 * H, Hp, dtype=torch.float32, device=dev)
        bias = []
        for d, s in enumerate(sfx):
            wih[d * 4 * H:(d + 1) * 4 * H, :isz] = f32(getattr(p, f"weight_ih_l{k}{s}"))
            whh[d, :, :H] = f32(getattr(p, f"weight_hh_l{k}{s}"))
            bias.append(f32(getattr(p, f"bias_ih_l{k}{s}")) + f32(getattr(p, f"bias_hh_l{k}{s}")))
        return dict(wih=split_from(wih), whh=split_from(whh), b=torch.cat(bias).contiguous(), K=Kp)

    def _pack_linear(self, lin):
        f32, dev = self._f32, self._device
        N, K = lin.weight.shape
        w = torch.zeros(N, _pad4(K), dtype=torch.float32, device=dev)
        w[:, :K] = f32(lin.weight)
        return split_from(w), f32(lin.bias)

    def _pack(self):
        pk = dict(layers=[])
        m = self._rnn_module()
        H, ndir, P = self.hidden_size, self.ndir, self._output_size
        isz = self._rnn_idim
        for i in range(self.num_layers):
            if self.use_projection:
                lw = self._pack_lstm(getattr(m, f"{'birnn' if self.bidirectional else 'rnn'}{i}"), 0, isz if i == 0 else P)
                lw["proj"] = self._pack_linear(getattr(m, f"bt{i}"))
            else:
                lw = self._pack_lstm(m.nbrnn, i, isz if i == 0 else ndir * H)
            pk["layers"].append(lw)
        if not self.use_projection:
            pk["l_last"] = self._pack_linear(m.l_last)
        if hasattr(self, "_pack_vgg"):
            pk["vgg"] = self._pack_vgg()
        self._packed = pk
        return pk

    # ---------------------------------------------------------------- launches
    def _lstm_layer(self, w, x, T, B, lens32, tag):
        """One (B)LSTM layer over x split [2][B*T][K] -> y split [2][B*T][pad4(ndir*H)] (rows t >= len zero)."""
        H, ndir = self.hidden_size, self.ndir
        Hp, ldy, M = _pad4(H), _pad4(ndir * H), B * T
        G = ndir * 4 * H
        xg = self._buf("xg", (M, G))
        ops.linear(x, w["wih"], xg, bias=w["b"])
        hg = self._buf("hg", (ndir, B, 4 * H))
        h = self._buf("h", (2, ndir, B, Hp), zero=True)       # pad columns stay 0 (the kernel writes j < H only)
        c = self._buf("c", (ndir, B, H))
        y = self._buf(f"y{tag}", (2, M, ldy), zero=True)
        for s in range(T):
            if s > 0:   # h_{s-1} W_hh^T of both directions: the direction is the GEMM's batch-y index
                ops.gemm(B, 4 * H, Hp, h, ndir * B * Hp, Hp, w["whh"], ndir * 4 * H * Hp, Hp, hg, 4 * H, nby=ndir, sa=(0, B * Hp),
                         sb=(0, 4 * H * Hp), sc=(0, B * 4 * H))
            ops.call("espb_lstm_rec_step_f32", ops.ptr(xg), ops.ptr(hg), ops.ptr(lens32), s, B, T, H, Hp, ndir, ops.ptr(h), ndir * B * Hp,
                     ops.ptr(c), ops.ptr(y), M * ldy, ldy)
            _count()
        return y

    def _project(self, lin, y, B, T, Tin, sub, lens32, act, out=None, out_split=None):
        """Linear over the frames 0, sub, 2 sub, ... of y split [2][B*Tin][K] -> out [B][T][N] plain (tanh when act, rows t >= len 0) and
        its split copy [2][B*T][pad4(N)]."""
        wsp, b = lin
        N, K = wsp.shape[1], wsp.shape[2]
        M = B * T
        if out is None:
            out = self._buf("proj", (B, T, N))
        ops.gemm(T, N, K, y, y.shape[1] * y.shape[2], sub * K, wsp, N * K, K, out, N, bias=b, nby=B, sa=(0, Tin * K), sc=(0, T * N))
        if out_split is None:
            out_split = self._buf("xs", (2, M, _pad4(N)), zero=True)
        ops.call("espb_rnn_proj_post_f32", ops.ptr(out), B, T, N, ops.ptr(lens32), 1 if act else 0, 1, ops.ptr(out_split), M * out_split.shape[2],
                 out_split.shape[2])
        _count()
        return out, out_split

    def _rnn(self, x, B, T, lens):
        """RNNP / RNN over x split [2][B*T][K] with per-utterance lengths lens (int64 CPU) -> (out (B, T', P), olens)."""
        pk, P, dev = self._packed, self._output_size, x.device
        subs = self._subsample
        out = None
        for i, w in enumerate(pk["layers"]):
            lens32 = lens.to(device=dev, dtype=torch.int32)
            y = self._lstm_layer(w, x, T, B, lens32, i % 2)
            if not self.use_projection:
                x = y
                continue
            sub = int(subs[i + 1]) if subs is not None else 1
            Tin = T
            if sub > 1:
                T = -(-T // sub)
                lens = (lens + 1) // sub
                lens32 = lens.to(device=dev, dtype=torch.int32)
            last = i + 1 == len(pk["layers"])
            if last:
                out = torch.empty(B, T, P, dtype=torch.float32, device=dev)
                split = self._buf("enc_split", (2, B * T, _pad4(P)), zero=True)
                out, x = self._project(w["proj"], y, B, T, Tin, sub, lens32, False, out=out, out_split=split)
            else:
                plain, x = self._project(w["proj"], y, B, T, Tin, sub, lens32, True)
            if self.trace is not None:
                self.trace.append((out if last else plain).clone())
        if not self.use_projection:
            lens32 = lens.to(device=dev, dtype=torch.int32)
            out = torch.empty(B, T, P, dtype=torch.float32, device=dev)
            split = self._buf("enc_split", (2, B * T, _pad4(P)), zero=True)
            out, x = self._project(pk["l_last"], x, B, T, T, 1, lens32, True, out=out, out_split=split)
        self.last_split_out = (out.data_ptr(), x) if P % 4 == 0 else None
        return out, lens

    @staticmethod
    def _packed_view(x, B, T, P):
        return (x[0] + x[1])[:, :P].reshape(B, T, P)

    def _check_input(self, xs_pad, ilens):
        ilens = torch.as_tensor(ilens).to("cpu", torch.int64)
        Tm = int(ilens.max())
        xs_pad = xs_pad[:, :Tm].contiguous().float()
        assert xs_pad.shape[2] == self.idim
        if int(ilens.min()) < 1:
            raise ValueError("espnet_b200 RNN encoders: every utterance needs at least one frame")
        return xs_pad, ilens


class VGGRNNEncoder(_RNNEncoderBase):
    """Drop-in for espnet2.asr.encoder.vgg_rnn_encoder.VGGRNNEncoder (inference, CUDA only)."""

    def __init__(self, input_size: int, rnn_type: str = "lstm", bidirectional: bool = True, use_projection: bool = True, num_layers: int = 4,
                 hidden_size: int = 320, output_size: int = 320, dropout: float = 0.0, in_channel: int = 1):
        super().__init__()
        self._init_common(input_size, rnn_type, bidirectional, use_projection, num_layers, hidden_size, output_size)
        if in_channel != 1:
            raise NotImplementedError(f"espnet_b200.VGGRNNEncoder implements in_channel 1 (got {in_channel})")
        self._rnn_idim = vgg2l_odim(input_size, in_channel)
        self._subsample = None
        rnn = (_RNNP if use_projection else _RNN)(self._rnn_idim, num_layers, hidden_size, output_size, bidirectional)
        self.enc = torch.nn.ModuleList([_VGG2L(in_channel), rnn])

    def _pack_vgg(self):
        f32, v = self._f32, self.enc[0]

        def gemm_w(cv):   # [co][ci][kt][kf] -> [co][(kt*3 + kf)*ci + c]
            co, ci = cv.weight.shape[:2]
            return split_from(f32(cv.weight).permute(0, 2, 3, 1).reshape(co, 9 * ci)), f32(cv.bias)

        return dict(c1_w=f32(v.conv1_1.weight).view(64, 9), c1_b=f32(v.conv1_1.bias), c12=gemm_w(v.conv1_2), c21=gemm_w(v.conv2_1),
                    c22=gemm_w(v.conv2_2))

    def _conv(self, a, w, B, F, T, Ci, Co, name):
        """3x3 stride-1 conv + ReLU over the zero-bordered split a [B][2][F+2][T+2][Ci] -> plain [B][F][T][Co]."""
        out = self._buf(name, (B, F, T, Co))
        ops.gemm(T, Co, 9 * Ci, a, 0, 0, w[0], Co * 9 * Ci, 9 * Ci, out, Co, bias=w[1], act=ACT_RELU, nbx=F, nby=B, sc=(T * Co, F * T * Co),
                 a_mode=2, conv=(T + 2, F + 2, Ci))
        return out

    def _vgg(self, xs, lens):
        """VGG2L (encoders.py VGG2L.forward) of xs (B, T, F) -> split rows [2][B*T4][128*F4] and the lengths after the two pools."""
        pk = self._packed["vgg"]
        B, T, F = xs.shape
        dev = xs.device
        l1 = lens.to(device=dev, dtype=torch.int32)
        lens2 = (lens + 1) // 2
        l2 = lens2.to(device=dev, dtype=torch.int32)
        T2, F2 = -(-T // 2), -(-F // 2)
        T4, F4 = -(-T2 // 2), -(-F2 // 2)
        a = self._buf("v_a", (B, 2, F + 2, T + 2, 64))
        ops.call("espb_vgg_conv1_relu_f32", ops.ptr(xs), B, T, F, ops.ptr(l1), ops.ptr(pk["c1_w"]), ops.ptr(pk["c1_b"]), 64, ops.ptr(a), T)
        _count()
        c = self._conv(a, pk["c12"], B, F, T, 64, 64, "v_c12")
        a = self._buf("v_p1", (B, 2, F2 + 2, T2 + 2, 64))
        ops.call("espb_vgg_pool_f32", ops.ptr(c), B, F, T, 64, ops.ptr(l1), 1, 0, ops.ptr(a), (F2 + 2) * (T2 + 2) * 64)
        _count()
        c = self._conv(a, pk["c21"], B, F2, T2, 64, 128, "v_c21")
        a = self._buf("v_p2", (B, 2, F2 + 2, T2 + 2, 128))
        ops.call("espb_vgg_pool_f32", ops.ptr(c), B, F2, T2, 128, ops.ptr(l2), 0, 0, ops.ptr(a), (F2 + 2) * (T2 + 2) * 128)
        _count()
        c = self._conv(a, pk["c22"], B, F2, T2, 128, 128, "v_c22")
        K = 128 * F4
        x = self._buf("v_out", (2, B * T4, K))
        ops.call("espb_vgg_pool_f32", ops.ptr(c), B, F2, T2, 128, ops.ptr(l2), 1, 1, ops.ptr(x), B * T4 * K)
        _count()
        return x, T4, (lens2 + 1) // 2

    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """xs_pad (B, T_f, idim) float32 CUDA, ilens (B,) -> (B, T, output_size), olens, None; rows t >= olens[b] are 0."""
        if prev_states is not None:
            raise NotImplementedError("espnet_b200.VGGRNNEncoder: prev_states (streaming) is not supported")
        self._packed or self._pack()
        xs, lens = self._check_input(xs_pad, ilens)
        x, T, lens = self._vgg(xs, lens)
        if self.trace is not None:
            self.trace.append(self._packed_view(x, xs.shape[0], T, x.shape[2]).clone())
        out, olens = self._rnn(x, xs.shape[0], T, lens)
        return out, olens, None


class RNNEncoder(_RNNEncoderBase):
    """Drop-in for espnet2.asr.encoder.rnn_encoder.RNNEncoder (inference, CUDA only)."""

    def __init__(self, input_size: int, rnn_type: str = "lstm", bidirectional: bool = True, use_projection: bool = True, num_layers: int = 4,
                 hidden_size: int = 320, output_size: int = 320, dropout: float = 0.0, subsample: Optional[Sequence[int]] = (2, 2, 1, 1)):
        super().__init__()
        self._init_common(input_size, rnn_type, bidirectional, use_projection, num_layers, hidden_size, output_size)
        if subsample is None:
            sub = [1] * (num_layers + 1)
        else:   # rnn_encoder.py: subsample[:num_layers], a 1 prepended, padded with 1 to num_layers + 1 entries
            sub = [1] + [int(s) for s in list(subsample)[:num_layers]]
            sub += [1] * (num_layers + 1 - len(sub))
        self._subsample = sub if use_projection else None
        self._rnn_idim = input_size
        rnn = (_RNNP if use_projection else _RNN)(input_size, num_layers, hidden_size, output_size, bidirectional)
        self.enc = torch.nn.ModuleList([rnn])

    @torch.no_grad()
    def forward(self, xs_pad: torch.Tensor, ilens: torch.Tensor, prev_states: torch.Tensor = None
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """xs_pad (B, T_f, idim) float32 CUDA, ilens (B,) -> (B, T, output_size), olens, None; rows t >= olens[b] are 0."""
        if prev_states is not None:
            raise NotImplementedError("espnet_b200.RNNEncoder: prev_states (streaming) is not supported")
        self._packed or self._pack()
        xs, lens = self._check_input(xs_pad, ilens)
        B, T, F = xs.shape
        Kp = _pad4(F)
        x = self._buf("in_split", (2, B * T, Kp), zero=True)
        ops.call("espb_rnn_proj_post_f32", ops.ptr(xs), B, T, F, ops.ptr(lens.to(device=xs.device, dtype=torch.int32)), 0, 0, ops.ptr(x),
                 B * T * Kp, Kp)
        _count()
        out, olens = self._rnn(x, B, T, lens)
        return out, olens, None
