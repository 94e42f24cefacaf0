"""TransformerLM and SequentialRNNLM (LSTM cells) as device-side incremental scorers for LM shallow fusion (SURVEY.md 8f-3).

Reference: espnet2/lm/transformer_lm.py:13-133 (embed -> legacy Encoder(input_layer="linear") -> Linear -> log_softmax; ``batch_score`` with a
per-layer cache of layer outputs), legacy/nets/pytorch_backend/transformer/encoder.py:132-139,366-392, encoder_layer.py:65-126, wired into the
search at espnet2/bin/asr_inference.py:178-191 (``scorers["lm"] = lm.lm``, weight ``lm_weight``).  Same constructor keywords and parameter
names, so a reference LM checkpoint (``ESPnetLanguageModel`` state_dict, keys ``lm.*``) loads by name.

Like the decoder (decoder.py) the new token of every hypothesis is scored against a position-major K / V cache addressed through the search's
ancestor table, instead of re-running the prefix: the decode-step kernels without the cross-attention.

Each LM also runs whole sentences (``forward`` / ``_logits``: the reference's forward, with the causal token-masked attention of
transformer_lm.py:57-72 for the TransformerLM), and ``ESPnetLanguageModel`` computes their negative log-likelihood for perplexity.

Limit: the reference masks prefix positions that hold token id 0 (``_target_mask``, transformer_lm.py:59-62: id 0 is the padding / blank id);
beam hypotheses never contain it in joint or CTC decoding (the CTC prefix score of blank is log-zero) -- a hypothesis with an explicit token 0
in attention-only decoding would be scored without that mask here.
"""
import math
from typing import Any, List, Tuple

import torch

from . import ops
from .decoder import KVCacheScorer, ScorerProtocol
from .layers import LN_EPS, _FFN, _MHA, PackedModule, _pitch
from .lib import call, ptr
from .ops import ACT_RELU, _count, layernorm, linear, split_from


class _LMLayer(torch.nn.Module):
    def __init__(self, d, units):
        super().__init__()
        self.self_attn = _MHA(d)
        self.feed_forward = _FFN(d, units)
        self.norm1 = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm2 = torch.nn.LayerNorm(d, eps=LN_EPS)


class _LMEncoder(torch.nn.Module):
    def __init__(self, idim, d, units, layers):
        super().__init__()
        # Sequential(Linear, LayerNorm(eps 1e-5), Dropout, ReLU, pos_enc): only indices 0 and 1 hold parameters
        self.embed = torch.nn.Sequential(torch.nn.Linear(idim, d), torch.nn.LayerNorm(d), torch.nn.Identity(), torch.nn.ReLU(), torch.nn.Identity())
        self.encoders = torch.nn.ModuleList(_LMLayer(d, units) for _ in range(layers))
        self.after_norm = torch.nn.LayerNorm(d, eps=LN_EPS)


class TransformerLM(KVCacheScorer):
    """Drop-in container for espnet2.lm.transformer_lm.TransformerLM (inference scorer)."""

    def __init__(self, vocab_size: int, pos_enc: str = None, embed_unit: int = 128, att_unit: int = 256, head: int = 2, unit: int = 1024,
                 layer: int = 4, dropout_rate: float = 0.1, positional_dropout_rate: float = 0.1, attention_dropout_rate: float = 0.1):
        super().__init__()
        if pos_enc not in (None, "sinusoidal"):
            raise ValueError(f"unknown pos-enc option: {pos_enc}")
        if att_unit // head > 128:
            raise NotImplementedError(f"espnet_b200 TransformerLM: attention head size <= 128 (got {att_unit} / {head} heads)")
        self.vocab_size, self.pos_enc, self.d, self.heads, self.units, self.num_blocks, self.embed_unit = (
            vocab_size, pos_enc, att_unit, head, unit, layer, embed_unit)
        self.embed = torch.nn.Embedding(vocab_size, embed_unit)
        self.encoder = _LMEncoder(embed_unit, att_unit, unit, layer)
        self.decoder = torch.nn.Linear(att_unit, vocab_size)

    def _pack(self):
        f32, e = self._f32, self.encoder
        pk = dict(emb=f32(self.embed.weight), in_w=split_from(f32(e.embed[0].weight)), in_b=f32(e.embed[0].bias),
                  in_ln=(*self._pack_ln(e.embed[1]), float(e.embed[1].eps)), layers=[])
        for lyr in e.encoders:
            pk["layers"].append(dict(**self._pack_mha(lyr.self_attn), n1=self._pack_ln(lyr.norm1), n2=self._pack_ln(lyr.norm2),
                                     ffn=self._pack_ffn(lyr.feed_forward)))
        pk["an"] = self._pack_ln(e.after_norm)
        pk["out_w"], pk["out_b"] = split_from(f32(self.decoder.weight)), f32(self.decoder.bias)
        self._packed = pk
        return pk

    def _iface_state(self, xs, n, need_len):
        st = getattr(self, "_iface_st", None)
        if st is None or st["n"] != n or st["max_len"] < need_len:
            st = self._iface_st = self.init_cache(n, max(32, 1 << (need_len - 1).bit_length()))
        return st

    # ---------------------------------------------------------------- device-side incremental scorer
    @torch.no_grad()
    def init_cache(self, n_slots, max_len):
        if self._packed is None:
            self._pack()
        L, D = self.num_blocks, self.d
        pe = self._pe(max_len) if self.pos_enc == "sinusoidal" else None
        return dict(n=n_slots, max_len=max_len, kc=self._buf("kc", (L, max_len, n_slots, D)), vc=self._buf("vc", (L, max_len, n_slots, D)), pe=pe)

    @torch.no_grad()
    def step(self, st, pos, last_tok, anc, step_ptr=None):
        """One position for all n slots: log-probabilities [n][V] of the next token (buffer reused across steps).  Equivalent of
        batch_score (transformer_lm.py:95-133) for prefixes whose newest token is ``last_tok`` at position ``pos`` (+ *step_ptr)."""
        pk = self._packed
        n, D, E = st["n"], self.d, self.embed_unit
        es = self._buf("es", (2, n, E))
        x = self._buf("x", (n, D))
        xn = self._buf("xn", (2, n, D))
        ctx = self._buf("ctx", (2, n, D))
        call("espb_gather_rows_split_f32", ptr(last_tok), ptr(pk["emb"]), n, E, ptr(es), n * E)
        _count()
        linear(es, pk["in_w"], x, bias=pk["in_b"])
        layernorm(x, pk["in_ln"][0], pk["in_ln"][1], pk["in_ln"][2], out_plain=x)
        call("espb_relu_posenc_f32", ptr(x), n, D, ptr(st["pe"]), pos, ptr(step_ptr), math.sqrt(D))
        _count()
        for li, w in enumerate(pk["layers"]):
            self._self_attn(x, xn, ctx, w, li, st, pos, anc, step_ptr)
            self._ffn(x, xn, w["n2"], w["ffn"], ACT_RELU)
        return self._head(x, xn, n)

    # ---------------------------------------------------------------- full-sequence forward (perplexity)
    def forward(self, input: torch.Tensor, hidden: None) -> Tuple[torch.Tensor, None]:
        """transformer_lm.py:62-72: logits (B, L, V) of every position of input (B, L), keys masked by _target_mask (token id 0 and the
        future)."""
        return _forward_logits(self, input), None

    @torch.no_grad()
    def _logits(self, tok, lens32, B, T):
        """Logits [B*T][V] (workspace) of token ids tok (B, T) int32 on the device: embedding, embed Linear + LayerNorm + ReLU (+ sinusoidal
        positions), the layers with causal attention, after_norm, output projection.  Rows t >= lens32[b] are not defined."""
        pk = self._packed or self._pack()
        D, E, M = self.d, self.embed_unit, B * T
        es = self._buf("es", (2, M, E))
        x = self._buf("x", (M, D))
        xn = self._buf("xn", (2, M, D))
        ctx = self._buf("ctx", (2, M, D))
        qkv = self._buf("qkv", (2, M, 3 * D))
        ops.call("espb_gather_rows_split_f32", ops.ptr(tok), ops.ptr(pk["emb"]), M, E, ops.ptr(es), M * E)
        _count()
        linear(es, pk["in_w"], x, bias=pk["in_b"])
        layernorm(x, pk["in_ln"][0], pk["in_ln"][1], pk["in_ln"][2], out_plain=x)
        ops.call("espb_relu_posenc_f32", ops.ptr(x), M, D, None, 0, None, 1.0)   # ReLU
        _count()
        if self.pos_enc == "sinusoidal":   # PositionalEncoding: x * sqrt(D) + pe[t], each product rounded like the reference's
            pe = self._pe(max(32, 1 << (T - 1).bit_length()))   # rows 0..T-1 of a power-of-two table: one table serves many lengths
            for b in range(B):
                xb = x[b * T:(b + 1) * T]
                ops.call("espb_axpby_f32", ops.ptr(xb), math.sqrt(D), ops.ptr(pe), 1.0, ops.ptr(xb), T * D)
            _count(B)
        for w in pk["layers"]:
            layernorm(x, *w["n1"], LN_EPS, out_split=xn)
            linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"], split_out=True)
            self._causal_attn(qkv, ctx, tok, lens32, B, T)
            linear(ctx, w["out_w"], x, bias=w["out_b"], residual=x)
            self._ffn(x, xn, w["n2"], w["ffn"], ACT_RELU)
        layernorm(x, *pk["an"], LN_EPS, out_split=xn)
        logits = self._buf("logits", (M, self.vocab_size))
        linear(xn, pk["out_w"], logits, bias=pk["out_b"])
        return logits

    def _causal_attn(self, qkv, ctx, tok, lens32, B, T):
        """Causal self-attention with the token-0 key mask, from the fused q|k|v projection qkv (split [2][B*T][3D]) to ctx (split
        [2][B*T][D]): the fused wgmma kernel for d_k = 64, else q k^T GEMM, masked softmax, p v GEMM."""
        D, H = self.d, self.heads
        dk, M, Tp = D // H, B * T, _pitch(T)
        vt = self._buf("vt", (2, B, H, dk, Tp))
        ops.call("espb_v_transpose_f32", ops.ptr(qkv), M * 3 * D, B, T, D, H, ops.ptr(lens32), ops.ptr(vt), B * H * dk * Tp, Tp)
        _count()
        if ops.use_flash_attn(dk):
            ops.call("espb_causal_flash_attn_f32", ops.ptr(qkv), 0, M * 3 * D, 3 * D, ops.ptr(qkv), D, M * 3 * D, 3 * D, ops.ptr(vt),
                     B * H * dk * Tp, Tp, ops.ptr(tok), ops.ptr(lens32), B, H, T, dk, ops.ptr(ctx), M * D, D)
            _count()
            return
        sc, probs = self._buf("sc", (B, H, T, Tp)), self._buf("probs", (2, B, H, T, Tp))
        ops.gemm(T, T, dk, qkv, M * 3 * D, 3 * D, qkv, M * 3 * D, 3 * D, sc, Tp, nbx=H, nby=B, sa=(dk, T * 3 * D), sb=(dk, T * 3 * D),
                 sc=(T * Tp, H * T * Tp), b_off=D)
        ops.call("espb_causal_softmax_f32", ops.ptr(sc), B, H, T, Tp, ops.ptr(lens32), ops.ptr(tok), math.sqrt(dk), ops.ptr(probs),
                 B * H * T * Tp)
        _count()
        ops.gemm(T, dk, T, probs, B * H * T * Tp, Tp, vt, B * H * dk * Tp, Tp, ctx, D, c_plane=M * D, split_out=True, nbx=H, nby=B,
                 sa=(T * Tp, H * T * Tp), sb=(dk * Tp, H * dk * Tp), sc=(dk, T * D))


def _forward_logits(lm, input):
    """forward(input, None) of either LM: every position of every row of input (B, L) is valid; a fresh (B, L, V) tensor."""
    input = torch.as_tensor(input)
    B, T = input.shape
    if B == 0 or T == 0:
        return torch.zeros(B, T, lm.vocab_size, dtype=torch.float32, device=lm._device)
    tok = _check_ids(input, lm.vocab_size).to(device=lm._device, dtype=torch.int32).contiguous()
    lens32 = torch.full((B,), T, dtype=torch.int32, device=tok.device)
    with _ws_tag(lm, "seq"):
        return lm._logits(tok, lens32, B, T).view(B, T, -1).clone()


def _check_ids(ids, V):
    if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= V):
        raise IndexError(f"token ids must lie in [0, {V}) (got {int(ids.min())} .. {int(ids.max())})")
    return ids


class _ws_tag:
    """Runs the full-sequence forward in a workspace set of its own, so that it neither reallocates nor overwrites the step scorer's."""

    def __init__(self, m, tag):
        self.m, self.tag = m, tag

    def __enter__(self):
        self.prev, self.m.ws_tag = self.m.ws_tag, self.tag

    def __exit__(self, *exc):
        self.m.ws_tag = self.prev


def _pad4(k):
    return (k + 3) & ~3


class _RNNParams(torch.nn.Module):
    """Holds nn.LSTM's parameters under nn.LSTM's names (weight_ih_l{k}, weight_hh_l{k}, bias_ih_l{k}, bias_hh_l{k}) without being an nn.LSTM:
    nn.LSTM re-flattens its weights through cuDNN when it moves to the GPU."""

    def __init__(self, ninp, nhid, nlayers):
        super().__init__()
        for k in range(nlayers):
            isz = ninp if k == 0 else nhid
            self.register_parameter(f"weight_ih_l{k}", torch.nn.Parameter(torch.empty(4 * nhid, isz)))
            self.register_parameter(f"weight_hh_l{k}", torch.nn.Parameter(torch.empty(4 * nhid, nhid)))
            self.register_parameter(f"bias_ih_l{k}", torch.nn.Parameter(torch.empty(4 * nhid)))
            self.register_parameter(f"bias_hh_l{k}", torch.nn.Parameter(torch.empty(4 * nhid)))
        bound = 1.0 / math.sqrt(nhid)   # nn.LSTM.reset_parameters
        for p in self.parameters():
            torch.nn.init.uniform_(p, -bound, bound)


class SequentialRNNLM(ScorerProtocol, PackedModule):
    """Drop-in container for espnet2.lm.seq_rnn_lm.SequentialRNNLM (inference scorer), LSTM cells only.

    One step for n hypotheses is 2L + 3 launches: one gather (embedding row and every layer's parent h into the GEMM operands), per layer one
    GEMM [input | parent h] @ [W_ih | W_hh]^T + (b_ih + b_hh) and one cell kernel, then the output projection and log-softmax.  The recurrent
    state lives in a two-deep ring h, c [2][L][n][Hp] addressed through the search's ancestor table, so it does not grow with the prefix.
    K of every GEMM is padded to a multiple of 4 (TMA needs 16-byte strides) with zero columns in weights and operands."""

    zero_bufs = True   # the operands' pad columns are zeroed when the buffers are created and never written afterwards

    def __init__(self, vocab_size: int, unit: int = 650, nhid: int = None, nlayers: int = 2, dropout_rate: float = 0.0, tie_weights: bool = False,
                 rnn_type: str = "lstm", ignore_id: int = 0):
        super().__init__()
        if nhid is None:
            nhid = unit
        rnn_type = rnn_type.upper()
        if rnn_type in ("GRU", "RNN_TANH", "RNN_RELU"):
            raise NotImplementedError(f"espnet_b200.SequentialRNNLM implements rnn_type lstm (got {rnn_type})")
        if rnn_type != "LSTM":
            raise ValueError("An invalid option for `--model` was supplied, options are ['LSTM', 'GRU', 'RNN_TANH' or 'RNN_RELU']")
        self.encoder = torch.nn.Embedding(vocab_size, unit, padding_idx=ignore_id)
        self.rnn = _RNNParams(unit, nhid, nlayers)
        self.decoder = torch.nn.Linear(nhid, vocab_size)
        if tie_weights:
            if nhid != unit:
                raise ValueError("When using the tied flag, nhid must be equal to emsize")
            self.decoder.weight = self.encoder.weight
        self.vocab_size, self.unit, self.nhid, self.nlayers, self.rnn_type = vocab_size, unit, nhid, nlayers, rnn_type

    def _pack(self):
        f32, dev = self._f32, self._device
        E, H, Ep, Hp = self.unit, self.nhid, _pad4(self.unit), _pad4(self.nhid)
        pk = dict(emb=f32(self.encoder.weight), layers=[])
        for k in range(self.nlayers):
            ip, isz = (Ep, E) if k == 0 else (Hp, H)
            w = torch.zeros(4 * H, ip + Hp, dtype=torch.float32, device=dev)
            w[:, :isz] = f32(getattr(self.rnn, f"weight_ih_l{k}"))
            w[:, ip:ip + H] = f32(getattr(self.rnn, f"weight_hh_l{k}"))
            pk["layers"].append((split_from(w), f32(getattr(self.rnn, f"bias_ih_l{k}")) + f32(getattr(self.rnn, f"bias_hh_l{k}"))))
        wo = torch.zeros(self.vocab_size, Hp, dtype=torch.float32, device=dev)
        wo[:, :H] = f32(self.decoder.weight)
        pk["out_w"], pk["out_b"] = split_from(wo), f32(self.decoder.bias)
        self._packed = pk
        return pk

    # ---------------------------------------------------------------- device-side incremental scorer
    @torch.no_grad()
    def init_cache(self, n_slots, max_len):
        """State of n_slots hypotheses; the ring does not depend on max_len."""
        if self._packed is None:
            self._pack()
        L, Hp = self.nlayers, _pad4(self.nhid)
        return dict(n=n_slots, h=self._buf("h", (2, L, n_slots, Hp)), c=self._buf("c", (2, L, n_slots, Hp)))

    @torch.no_grad()
    def step(self, st, pos, last_tok, anc, step_ptr=None):
        """One position for all n slots: log-probabilities [n][V] of the next token (buffer reused across steps).  Equivalent of batch_score
        (seq_rnn_lm.py:127-166) for hypotheses whose newest token is ``last_tok`` at position ``pos`` (+ *step_ptr) and whose parent state is
        ring (pos-1)&1 at slot anc[s][pos-1]."""
        pk = self._packed
        n, L, E, H = st["n"], self.nlayers, self.unit, self.nhid
        Ep, Hp = _pad4(E), _pad4(H)
        kp0, kp1 = Ep + Hp, 2 * Hp
        xs = self._buf("xs", (2 * n * kp0 + 2 * (L - 1) * n * kp1,))
        xo = self._buf("xo", (2, n, Hp))
        gates = self._buf("gates", (n, 4 * H))
        ops_ = [xs[:2 * n * kp0].view(2, n, kp0)] + [xs[2 * n * kp0 + 2 * l * n * kp1:2 * n * kp0 + 2 * (l + 1) * n * kp1].view(2, n, kp1)
                                                       for l in range(L - 1)]
        call("espb_rnnlm_gather_f32", ptr(last_tok), ptr(pk["emb"]), E, Ep, ptr(anc), anc.shape[1], pos, ptr(step_ptr), ptr(st["h"]), L, n, H, Hp,
             ptr(xs))
        _count()
        for li, (w, b) in enumerate(pk["layers"]):
            linear(ops_[li], w, gates, bias=b)
            nxt = ops_[li + 1] if li + 1 < L else xo
            call("espb_lstm_cell_f32", ptr(gates), ptr(anc), anc.shape[1], pos, ptr(step_ptr), ptr(st["h"]), ptr(st["c"]), li, L, n, H, Hp,
                 ptr(nxt), nxt[0].numel(), nxt.shape[2])
            _count()
        logp = self._buf("logp", (n, self.vocab_size))
        linear(xo, pk["out_w"], logp, bias=pk["out_b"])
        ops.log_softmax_rows_(logp)
        return logp

    # ---------------------------------------------------------------- full-sequence forward (perplexity)
    def forward(self, input: torch.Tensor, hidden: None) -> Tuple[torch.Tensor, None]:
        """seq_rnn_lm.py:84-96 from the zero state: logits (B, L, V) of every position of input (B, L).  The final (h, c) is not returned
        (None), and a given hidden state is refused."""
        if hidden is not None:
            raise NotImplementedError("espnet_b200 SequentialRNNLM.forward starts from the zero state (hidden=None)")
        return _forward_logits(self, input), None

    @torch.no_grad()
    def _logits(self, tok, lens32, B, T):
        """Logits [B*T][V] (workspace) of token ids tok (B, T) int32 on the device.  Per layer one GEMM of the inputs of all positions with
        W_ih (+ both biases), then per step h W_hh^T and the cell (espb_lstm_rec_step_f32); utterance b stops at lens32[b] (its rows past
        it are 0, as the padded steps of a unidirectional LSTM never reach the valid ones)."""
        pk = self._packed or self._pack()
        E, H, L, M = self.unit, self.nhid, self.nlayers, B * T
        Ep, Hp = _pad4(E), _pad4(H)
        kp0 = Ep + Hp
        # layer 0's operand in the step layout [embedding | zero h] (pitch Ep + Hp, 16-byte rows for TMA); the K = Ep GEMM reads the
        # embedding half.  The layer outputs alternate between two buffers; y[0] stands in for the h ring the gather does not read at pos 0.
        xs = self._buf("seq_x0", (2, M, kp0), zero=True)
        ys = [self._buf(f"seq_y{i}", (2, M, Hp), zero=True) for i in range(min(L, 2))]
        ops.call("espb_rnnlm_gather_f32", ops.ptr(tok), ops.ptr(pk["emb"]), E, Ep, None, 0, 0, None, ops.ptr(ys[0]), 1, M, H, Hp, ops.ptr(xs))
        _count()
        xg, hg = self._buf("seq_xg", (M, 4 * H)), self._buf("seq_hg", (B, 4 * H))
        h, c = self._buf("seq_h", (2, B, Hp), zero=True), self._buf("seq_c", (B, H))
        for li, (w, bias) in enumerate(pk["layers"]):
            ip = Ep if li == 0 else Hp
            kp = ip + Hp
            x, lda = (xs, kp0) if li == 0 else (ys[(li - 1) % 2], Hp)
            y = ys[li % 2]
            ops.gemm(M, 4 * H, ip, x, M * lda, lda, w, 4 * H * kp, kp, xg, 4 * H, bias=bias)
            for s in range(T):
                if s > 0:   # h_{s-1} W_hh^T: the recurrent half of the packed [W_ih | W_hh]
                    ops.gemm(B, 4 * H, Hp, h, B * Hp, Hp, w, 4 * H * kp, kp, hg, 4 * H, b_off=ip)
                ops.call("espb_lstm_rec_step_f32", ops.ptr(xg), ops.ptr(hg), ops.ptr(lens32), s, B, T, H, Hp, 1, ops.ptr(h), B * Hp, ops.ptr(c),
                         ops.ptr(y), M * Hp, Hp)
                _count()
        logits = self._buf("logits", (M, self.vocab_size))
        linear(ys[(L - 1) % 2], pk["out_w"], logits, bias=pk["out_b"])
        return logits

    # ---------------------------------------------------------------- BatchScorerInterface (scorer_interface.py:85-188): per hypothesis (h, c)
    @torch.no_grad()
    def batch_score(self, ys: torch.Tensor, states: List[Any], xs: torch.Tensor) -> Tuple[torch.Tensor, List[Any]]:
        """seq_rnn_lm.py:127-166: states per hypothesis (h, c), each [nlayers, nhid], or None at the start (zero state)."""
        n = ys.shape[0]
        self.ws_tag = "iface"
        st = getattr(self, "_iface_st", None)
        if st is None or st["n"] != n or self._packed is None:
            st = self._iface_st = self.init_cache(n, 1)
        H = self.nhid
        pos = 0 if states[0] is None else 1
        if pos:     # parents in ring 0, slot s = hypothesis s
            st["h"][0, :, :, :H] = torch.stack([s[0] for s in states], dim=1)
            st["c"][0, :, :, :H] = torch.stack([s[1] for s in states], dim=1)
        anc = self._buf("iface_anc", (n, 1), dtype=torch.int32)
        anc.copy_(torch.arange(n, dtype=torch.int32, device=anc.device).view(n, 1))
        logp = self.step(st, pos, ys[:, -1].to(torch.int32).contiguous(), anc, None)
        h, c = st["h"][pos & 1, :, :, :H], st["c"][pos & 1, :, :, :H]
        return logp.clone(), [(h[:, b].clone(), c[:, b].clone()) for b in range(n)]


def build_lm_from_file(config_file, model_file=None, device="cuda"):
    """LMTask.build_model_from_file (espnet2/tasks/lm.py, abs_task.py:2456-2561) for ``lm: transformer`` and ``lm: seq_rnn`` (the default when
    the config has no ``lm`` key): yaml -> TransformerLM / SequentialRNNLM -> weights (checkpoint keys carry the ``lm.`` prefix of
    ESPnetLanguageModel)."""
    import argparse

    import yaml

    with open(config_file, "r", encoding="utf-8") as f:
        args = argparse.Namespace(**yaml.safe_load(f))
    classes = dict(transformer=TransformerLM, seq_rnn=SequentialRNNLM)
    kind = getattr(args, "lm", None) or "seq_rnn"
    if kind not in classes:
        raise NotImplementedError(f"espnet_b200 implements lm: transformer and lm: seq_rnn (got {kind!r})")
    lm = classes[kind](vocab_size=len(args.token_list), **(getattr(args, "lm_conf", None) or {}))
    if model_file is not None:
        sd = torch.load(model_file, map_location="cpu")
        lm.load_state_dict({k[3:]: v for k, v in sd.items() if k.startswith("lm.")}, strict=True)
    return lm.to(device).eval(), args


class ESPnetLanguageModel(torch.nn.Module):
    """Drop-in container for espnet2.lm.espnet_model.ESPnetLanguageModel (inference): ``lm`` (so the checkpoint keys are ``lm.*``), sos = eos =
    vocab_size - 1, ``nll`` and ``batchify_nll``.  The negative log-likelihood runs on the device: the LM's full-sequence logits, then one
    kernel that reads each logit row once (espb_nll_rows_f32)."""

    def __init__(self, lm: torch.nn.Module, vocab_size: int, ignore_id: int = 0):
        super().__init__()
        if not isinstance(lm, (TransformerLM, SequentialRNNLM)):
            raise NotImplementedError(f"espnet_b200 ESPnetLanguageModel wraps TransformerLM and SequentialRNNLM (got {type(lm).__name__})")
        self.lm = lm
        self.sos = self.eos = vocab_size - 1
        self.ignore_id = ignore_id

    @torch.no_grad()
    def nll(self, text: torch.Tensor, text_lengths: torch.Tensor, max_length: int = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """espnet_model.py:24-70: x = <eos> text, t = text <sos>; nll (B, L + 1) with 0 at positions >= text_lengths + 1, and text_lengths + 1."""
        B = text.shape[0]
        lens = torch.as_tensor(text_lengths).cpu().long()
        text = text[:, : int(lens.max())] if max_length is None else text[:, : int(max_length)]
        T = text.shape[1] + 1
        x_lengths = torch.as_tensor(text_lengths) + 1
        dev = self.lm._device
        pos = torch.arange(T).view(1, T)
        valid = pos < (lens + 1).view(B, 1)                     # positions whose nll the reference keeps
        x = torch.zeros(B, T, dtype=torch.long)                 # positions past a sentence hold 0: they never reach a valid one
        x[:, 0] = self.eos
        x[:, 1:] = text.cpu()
        x = torch.where(valid, x, torch.zeros_like(x))
        tgt = torch.full((B, T), -1, dtype=torch.long)          # -1: written as 0 by the kernel
        tgt[:, :-1] = text.cpu()
        tgt[torch.arange(B), lens.clamp(max=T - 1)] = self.sos  # t[i, l] = sos
        tgt = torch.where(valid, tgt, torch.full_like(tgt, -1))
        if B == 0:
            return torch.zeros(0, T, device=dev), x_lengths
        _check_ids(x, self.lm.vocab_size)
        _check_ids(tgt[valid], self.lm.vocab_size)
        x32 = x.to(device=dev, dtype=torch.int32)
        t32 = tgt.to(device=dev, dtype=torch.int32)
        lens32 = (lens + 1).clamp(max=T).to(device=dev, dtype=torch.int32)
        out = torch.empty(B, T, dtype=torch.float32, device=dev)
        with _ws_tag(self.lm, "seq"):
            logits = self.lm._logits(x32, lens32, B, T)
            ops.call("espb_nll_rows_f32", ops.ptr(logits), B * T, logits.stride(0), self.lm.vocab_size, ops.ptr(t32), ops.ptr(out))
            _count()
        return out, x_lengths

    def batchify_nll(self, text: torch.Tensor, text_lengths: torch.Tensor, batch_size: int = 100) -> Tuple[torch.Tensor, torch.Tensor]:
        """espnet_model.py:72-114: nll in chunks of batch_size sentences, all padded to the longest."""
        total = text.size(0)
        if total <= batch_size:
            return self.nll(text, text_lengths)
        max_length = int(torch.as_tensor(text_lengths).max())
        nlls, x_lengths = [], []
        for start in range(0, total, batch_size):
            n, xl = self.nll(text[start:start + batch_size], text_lengths[start:start + batch_size], max_length=max_length)
            nlls.append(n)
            x_lengths.append(xl)
        return torch.cat(nlls), torch.cat(x_lengths)


def build_espnet_lm_from_file(config_file, model_file=None, device="cuda"):
    """LMTask.build_model_from_file returning the whole ESPnetLanguageModel (tasks/lm.py:173-210): build_lm_from_file's LM wrapped with the
    config's model_conf."""
    lm, args = build_lm_from_file(config_file, model_file, device)
    model = ESPnetLanguageModel(lm, vocab_size=len(args.token_list), **(getattr(args, "model_conf", None) or {}))
    return model.eval(), args
