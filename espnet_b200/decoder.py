"""TransformerDecoder with the reference's constructor / state_dict surface, as an incremental device-side
scorer: cross-attention K/V are projected once per utterance (shared by the whole beam) and the
self-attention K/V of each new token are appended to a position-major cache addressed through an
ancestor table, instead of re-projecting the prefix and the memory every step as the reference does.
``KVCacheScorer`` holds what the decoder and the Transformer LM (lm.py) share: the scorer protocol,
the sinusoid table, the self-attention block, the output head and the K/V-state ``batch_score``.

Reference: espnet2/asr/decoder/transformer_decoder.py:60-311, 413-470;
espnet2/legacy/nets/pytorch_backend/transformer/decoder_layer.py:73-179 (cache branch), attention.py:153-265
(default branch, no flash/sdpa), embedding.py:38-95 (PositionalEncoding).
"""
import math
from typing import List

import torch

from . import ops
from .layers import LN_EPS, _FFN, _MHA, PackedModule, abs_pos_table
from .lib import call, ptr
from .ops import ACT_RELU, _count, layernorm, linear, split_from


class ScorerProtocol:
    """The state handling of the reference's BatchScorerInterface (espnet2/legacy/nets/scorer_interface.py:85-188) for a scorer whose
    state is None at the start and, after a ``batch_score``, a list with one entry per hypothesis."""

    def init_state(self, x: torch.Tensor):
        return None

    def batch_init_state(self, x: torch.Tensor):
        return self.init_state(x)

    def select_state(self, state, i: int, new_id: int = None):
        return None if state is None else state[i]

    def final_score(self, state) -> float:
        return 0.0


class KVCacheScorer(ScorerProtocol, PackedModule):
    """A Transformer scorer that runs one position for n hypothesis slots per ``step`` over a self-attention K / V cache
    st["kc"], st["vc"] [L][max_len][n][D], the prefix of slot s being addressed through the search's ancestor table.  Subclasses set
    ``d`` and ``heads``, pack ``n1`` / ``qkv_*`` / ``out_*`` per layer and ``an`` / ``out_w`` / ``out_b``, and define ``step`` and
    ``_iface_state``.

    ``batch_score`` is the reference's functional protocol: a hypothesis' state is (k, v), the self-attention K / V rows of its prefix for
    every layer, each [L][len][D] (the reference keeps the layer OUTPUTS of the prefix and re-projects them every step).  Each call copies
    the states into the cache and runs the same kernels as the device-resident search (``step``); espnet_b200.BatchBeamSearch does not go
    through here."""

    def _pe(self, length):
        """Sinusoid table of positions 0..length-1 (PositionalEncoding), one per length."""
        key = ("pe", length)
        if key not in self._ws:
            self._ws[key] = abs_pos_table(length, self.d).to(self._device)
        return self._ws[key]

    def _self_attn(self, x, xn, ctx, w, li, st, pos, anc, step_ptr):
        """x += linear_out(self-attention of layer li (LN(x))): the new token's q / k / v in one GEMM, its k / v appended to the cache at
        position pos (+ *step_ptr), attention over the slot's prefix, then the output projection with the residual.  Launches through
        ops.call / ops.ptr, looked up at call time, like the shared code of layers.py: the kernel emulation of the tests replaces them in ops,
        whichever module the subclass lives in."""
        n, D = st["n"], self.d
        qkv = self._buf("qkv", (n, 3 * D))
        layernorm(x, *w["n1"], LN_EPS, out_split=xn)
        linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"])
        ops.call("espb_dec_self_attn_f32", ops.ptr(qkv), ops.ptr(st["kc"][li]), ops.ptr(st["vc"][li]), ops.ptr(anc), anc.shape[1], n, D,
                 self.heads, pos, ops.ptr(step_ptr), st["max_len"], ops.ptr(ctx), n * D)
        _count()
        linear(ctx, w["out_w"], x, bias=w["out_b"], residual=x)

    def _head(self, x, xn, n):
        """after_norm, output projection and log_softmax -> log-probabilities [n][V] (buffer reused across steps)."""
        pk = self._packed
        layernorm(x, *pk["an"], LN_EPS, out_split=xn)
        logp = self._buf("logp", (n, pk["out_w"].shape[1]))
        linear(xn, pk["out_w"], logp, bias=pk["out_b"])
        ops.log_softmax_rows_(logp)
        return logp

    @torch.no_grad()
    def batch_score(self, ys: torch.Tensor, states, xs: torch.Tensor):
        """ys (n, len) int64 prefixes (with sos), states: list of n per-hypothesis states (None at the first step), xs (n, T, D) the
        encoder output repeated per hypothesis -> (log-probabilities (n, V), list of n new states)."""
        n, ln = ys.shape
        pos = ln - 1
        self.ws_tag = "iface"
        st = self._iface_state(xs, n, ln)
        kc, vc = st["kc"], st["vc"]
        if pos > 0:
            kc[:, :pos] = torch.stack([s[0] for s in states], dim=2)
            vc[:, :pos] = torch.stack([s[1] for s in states], dim=2)
        anc = self._buf("iface_anc", (n, st["max_len"] + 1), dtype=torch.int32)
        anc.copy_(torch.arange(n, dtype=torch.int32, device=anc.device).view(n, 1).expand_as(anc))   # every slot is its own ancestor
        logp = self.step(st, pos, ys[:, -1].to(torch.int32).contiguous(), anc)
        return logp.clone(), [(kc[:, :ln, b].clone(), vc[:, :ln, b].clone()) for b in range(n)]


class _DecoderLayer(torch.nn.Module):
    def __init__(self, d, units):
        super().__init__()
        self.self_attn, self.src_attn = _MHA(d), _MHA(d)
        self.feed_forward = _FFN(d, units)
        self.norm1 = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm2 = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm3 = torch.nn.LayerNorm(d, eps=LN_EPS)


class TransformerDecoder(KVCacheScorer):
    """Drop-in container for espnet2.asr.decoder.transformer_decoder.TransformerDecoder (inference scorer)."""

    def __init__(self, vocab_size: int, encoder_output_size: int, attention_heads: int = 4, linear_units: int = 2048,
                 num_blocks: int = 6, dropout_rate: float = 0.1, positional_dropout_rate: float = 0.1,
                 self_attention_dropout_rate: float = 0.0, src_attention_dropout_rate: float = 0.0, input_layer: str = "embed",
                 use_output_layer: bool = True, pos_enc_class=None, normalize_before: bool = True, concat_after: bool = False,
                 layer_drop_rate: float = 0.0, qk_norm: bool = False, use_flash_attn: bool = True,
                 gradient_checkpoint_layers: List[int] = []):
        super().__init__()
        if input_layer != "embed" or not use_output_layer or not normalize_before or concat_after or qk_norm:
            raise NotImplementedError("espnet_b200 TransformerDecoder: embed input, output layer, pre-LN, no concat_after/qk_norm")
        d = encoder_output_size
        if d // attention_heads > 128:
            raise NotImplementedError(f"espnet_b200 TransformerDecoder: attention head size <= 128 (got {d} / {attention_heads} heads)")
        self.d, self.heads, self.units, self.num_blocks, self.odim = d, attention_heads, linear_units, num_blocks, vocab_size
        self.embed = torch.nn.Sequential(torch.nn.Embedding(vocab_size, d))
        self.decoders = torch.nn.ModuleList(_DecoderLayer(d, linear_units) for _ in range(num_blocks))
        self.after_norm = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.output_layer = torch.nn.Linear(d, vocab_size)

    def _pack(self):
        f32 = self._f32
        pk = dict(emb=f32(self.embed[0].weight), layers=[])
        kvw, kvb = [], []
        for lyr in self.decoders:
            ca = lyr.src_attn
            pk["layers"].append(dict(
                **self._pack_mha(lyr.self_attn), n1=self._pack_ln(lyr.norm1), n2=self._pack_ln(lyr.norm2), n3=self._pack_ln(lyr.norm3),
                cq_w=split_from(f32(ca.linear_q.weight)), cq_b=f32(ca.linear_q.bias),
                co_w=split_from(f32(ca.linear_out.weight)), co_b=f32(ca.linear_out.bias), ffn=self._pack_ffn(lyr.feed_forward)))
            kvw += [f32(ca.linear_k.weight), f32(ca.linear_v.weight)]
            kvb += [f32(ca.linear_k.bias), f32(ca.linear_v.bias)]
        pk["kv_w"], pk["kv_b"] = split_from(torch.cat(kvw, 0)), torch.cat(kvb, 0)  # [L*2D][D]: per layer k rows then v rows
        pk["an"] = self._pack_ln(self.after_norm)
        pk["out_w"], pk["out_b"] = split_from(f32(self.output_layer.weight)), f32(self.output_layer.bias)
        self._packed = pk
        return pk

    def _iface_state(self, xs, n, need_len):
        """Cross-attention K / V of the utterance whose encoder output is xs[0] (T, D): projected once and kept while it is the same
        tensor; the self-attention cache for n slots of at least need_len positions."""
        x = xs[0]
        key = (x.data_ptr(), tuple(x.shape), tuple(x.stride()), x._version)
        c = getattr(self, "_iface", None)
        if c is None or c["key"] != key:
            T = x.shape[0]
            # ``x_ref`` keeps the storage alive: while it is cached no other encoder output can be allocated at the same address, so an equal key
            # means the same data (a freed tensor's address is readily reused for the next utterance of the same length)
            c = self._iface = dict(key=key, x_ref=x, enc_split=split_from(x.contiguous().float()),
                                   lens32=torch.tensor([T], dtype=torch.int32, device=x.device), T=T, st=None)
        st = c["st"]
        if st is None or st["n"] != n or st["max_len"] < need_len:
            cap = max(32, 1 << (need_len - 1).bit_length())
            c["st"] = st = self.init_memory(c["enc_split"], 1, c["T"], c["lens32"], n, cap)
        return st

    @torch.no_grad()
    def score(self, ys: torch.Tensor, state, x: torch.Tensor):
        """ScorerInterface.score for one hypothesis (transformer_decoder.py:240-260)."""
        logp, states = self.batch_score(ys.unsqueeze(0), [state], x.unsqueeze(0))
        return logp[0], states[0]

    # ---------------------------------------------------------------- device-side incremental scorer
    @torch.no_grad()
    def init_memory(self, enc_split, U, Tmax, lens32, n_slots, max_len):
        """Project the encoder memory once per utterance (shared by the beam); allocate the self-attention cache.  Slot s belongs to
        utterance s // (n_slots / U)."""
        pk = self._packed or self._pack()
        L, D, H = self.num_blocks, self.d, self.heads
        dk = D // H
        # kvmem[l][0|1][u][h][t][dk]: one contiguous block per (layer, k/v, utterance, head) -> the per-step cross-attention streams it
        kvmem = self._buf("kvmem", (L, 2, U, H, Tmax, dk), zero=True)
        for l in range(L):
            for j in range(2):   # heads as batch-x (weight rows / bias / output block per head), utterances as batch-y
                ops.gemm(Tmax, dk, D, enc_split, U * Tmax * D, D, pk["kv_w"], L * 2 * D * D, D, kvmem, dk, bias=pk["kv_b"],
                         nbx=H, nby=U, sa=(0, Tmax * D), sb=(dk * D, 0), sc=(Tmax * dk, H * Tmax * dk), b_off=(l * 2 + j) * D * D,
                         c_off=(l * 2 + j) * U * H * Tmax * dk, sbias_x=dk, bias_off=(l * 2 + j) * D)
        st = dict(kvmem=kvmem, U=U, Tmax=Tmax, lens32=lens32, n=n_slots, W=n_slots // U, max_len=max_len,
                  kc=self._buf("kc", (L, max_len, n_slots, D)), vc=self._buf("vc", (L, max_len, n_slots, D)),
                  pe=self._pe(max_len))
        return st

    @torch.no_grad()
    def step(self, st, pos, last_tok, anc, step_ptr=None):
        """One decoding position for all n slots: returns log-probabilities [n][V] (buffer reused across steps).
        With ``step_ptr`` (device int32) the position is ``pos + *step_ptr`` so that a captured CUDA graph can be replayed.
        Equivalent of batch_score/forward_one_step (transformer_decoder.py:262-311,191-238)."""
        pk = self._packed
        n, D, H = st["n"], self.d, self.heads
        x = self._buf("x", (n, D))
        xn = self._buf("xn", (2, n, D))
        ctx = self._buf("ctx", (2, n, D))
        q = self._buf("q", (n, D))
        call("espb_dec_embed_f32", ptr(last_tok), ptr(pk["emb"]), ptr(st["pe"]), pos, ptr(step_ptr), n, D, math.sqrt(D), ptr(x))
        _count()
        for li, w in enumerate(pk["layers"]):
            self._self_attn(x, xn, ctx, w, li, st, pos, anc, step_ptr)
            layernorm(x, *w["n2"], LN_EPS, out_split=xn)
            linear(xn, w["cq_w"], q, bias=w["cq_b"])
            call("espb_dec_src_attn_f32", ptr(q), ptr(st["kvmem"][li, 0]), ptr(st["kvmem"][li, 1]), st["U"], st["Tmax"],
                 ptr(st["lens32"]), st["W"], D, H, ptr(ctx), n * D)
            _count()
            linear(ctx, w["co_w"], x, bias=w["co_b"], residual=x)
            self._ffn(x, xn, w["n3"], w["ffn"], ACT_RELU)
        return self._head(x, xn, n)
