"""TransformerDecoder with the reference's constructor / state_dict surface, as an incremental device-side
scorer: cross-attention K/V are projected once per utterance (shared by the whole beam) and the
self-attention K/V of each new token are appended to a position-major cache addressed through an
ancestor table, instead of re-projecting the prefix and the memory every step as the reference does.

Reference: espnet2/asr/decoder/transformer_decoder.py:60-311, 413-470;
espnet2/legacy/nets/pytorch_backend/transformer/decoder_layer.py:73-179 (cache branch), attention.py:153-265
(default branch, no flash/sdpa), embedding.py:38-95 (PositionalEncoding).
"""
import math
from typing import List

import torch

from . import ops
from .layers import LN_EPS, _FFN, _MHA, abs_pos_table
from .lib import call, ptr
from .ops import ACT_RELU, _count, layernorm, linear, new_split, split_from


class _DecoderLayer(torch.nn.Module):
    def __init__(self, d, units):
        super().__init__()
        self.self_attn, self.src_attn = _MHA(d), _MHA(d)
        self.feed_forward = _FFN(d, units)
        self.norm1 = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm2 = torch.nn.LayerNorm(d, eps=LN_EPS)
        self.norm3 = torch.nn.LayerNorm(d, eps=LN_EPS)


class TransformerDecoder(torch.nn.Module):
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
        self._packed = None
        self._ws = {}

    def _load_from_state_dict(self, *args, **kwargs):
        self._packed = None
        return super()._load_from_state_dict(*args, **kwargs)

    def _pack(self):
        dev = self.after_norm.weight.device
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        pk = dict(emb=f32(self.embed[0].weight), layers=[])
        kvw, kvb = [], []
        for lyr in self.decoders:
            sa, ca, ff = lyr.self_attn, lyr.src_attn, lyr.feed_forward
            d = dict(
                n1=(f32(lyr.norm1.weight), f32(lyr.norm1.bias)), n2=(f32(lyr.norm2.weight), f32(lyr.norm2.bias)),
                n3=(f32(lyr.norm3.weight), f32(lyr.norm3.bias)),
                qkv_w=split_from(torch.cat([f32(sa.linear_q.weight), f32(sa.linear_k.weight), f32(sa.linear_v.weight)], 0)),
                qkv_b=torch.cat([f32(sa.linear_q.bias), f32(sa.linear_k.bias), f32(sa.linear_v.bias)], 0),
                so_w=split_from(f32(sa.linear_out.weight)), so_b=f32(sa.linear_out.bias),
                cq_w=split_from(f32(ca.linear_q.weight)), cq_b=f32(ca.linear_q.bias),
                co_w=split_from(f32(ca.linear_out.weight)), co_b=f32(ca.linear_out.bias),
                w1=split_from(f32(ff.w_1.weight)), b1=f32(ff.w_1.bias), w2=split_from(f32(ff.w_2.weight)), b2=f32(ff.w_2.bias))
            kvw += [f32(ca.linear_k.weight), f32(ca.linear_v.weight)]
            kvb += [f32(ca.linear_k.bias), f32(ca.linear_v.bias)]
            pk["layers"].append(d)
        pk["kv_w"], pk["kv_b"] = split_from(torch.cat(kvw, 0)), torch.cat(kvb, 0)  # [L*2D][D]: per layer k rows then v rows
        pk["an"] = (f32(self.after_norm.weight), f32(self.after_norm.bias))
        pk["out_w"], pk["out_b"] = split_from(f32(self.output_layer.weight)), f32(self.output_layer.bias)
        self._packed = pk
        return pk

    ws_tag = 0   # workspace set in use: the search runs independent utterance groups on separate streams, each with its own buffers

    def _buf(self, name, shape, dtype=torch.float32, zero=False):
        name = (self.ws_tag, name)
        key = (name, tuple(shape), dtype)
        t = self._ws.get(key)
        if t is None:
            for k in [k for k in self._ws if k[0] == name]:
                del self._ws[k]
            t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=self.after_norm.weight.device)
            self._ws[key] = t
            self.buf_version = getattr(self, "buf_version", 0) + 1   # captured CUDA graphs hold these pointers
        return t

    # ---------------------------------------------------------------- BatchScorerInterface (espnet2/legacy/nets/scorer_interface.py:85-188)
    # The functional scorer protocol of the reference's (Batch)BeamSearch: states are opaque objects the search threads through
    # select_state / batch_score, so the reference's own search can drive this decoder.  A hypothesis' state is (k, v): the
    # self-attention K / V rows of its prefix for every layer, each [L][len][D] (the reference keeps the layer OUTPUTS of the
    # prefix, transformer_decoder.py:262-311, and re-projects them every step).  Each call copies the states into the position-major
    # cache and runs the same kernels as the device-resident search (`step`); espnet_b200.BatchBeamSearch does not go through here.
    def init_state(self, x: torch.Tensor):
        return None

    def batch_init_state(self, x: torch.Tensor):
        return self.init_state(x)

    def select_state(self, state, i: int, new_id: int = None):
        return None if state is None else state[i]

    def final_score(self, state) -> float:
        return 0.0

    def _iface_memory(self, x, n, need_len):
        """Cross-attention K / V of the utterance whose encoder output is x (T, D): projected once and kept while x is the same tensor."""
        key = (x.data_ptr(), tuple(x.shape), tuple(x.stride()), x._version)
        c = getattr(self, "_iface", None)
        if c is None or c["key"] != key:
            T = x.shape[0]
            self.ws_tag = "iface"
            # ``x_ref`` keeps the storage alive: while it is cached no other encoder output can be allocated at the same address, so an equal key
            # means the same data (a freed tensor's address is readily reused for the next utterance of the same length)
            c = self._iface = dict(key=key, x_ref=x, enc_split=split_from(x.contiguous().float()),
                                   lens32=torch.tensor([T], dtype=torch.int32, device=x.device), T=T, st=None)
        st = c["st"]
        if st is None or st["n"] != n or st["max_len"] < need_len:
            cap = max(32, 1 << (need_len - 1).bit_length())
            self.ws_tag = "iface"
            c["st"] = st = self.init_memory(c["enc_split"], 1, c["T"], c["lens32"], n, cap)
        return st

    @torch.no_grad()
    def batch_score(self, ys: torch.Tensor, states, xs: torch.Tensor):
        """ys (n, len) int64 prefixes (with sos), states: list of n per-hypothesis states (None at the first step), xs (n, T, D) the
        encoder output repeated per hypothesis -> (log-probabilities (n, V), list of n new states).  transformer_decoder.py:262-311."""
        n, ln = ys.shape
        pos = ln - 1
        st = self._iface_memory(xs[0], n, ln)
        self.ws_tag = "iface"
        L, D = self.num_blocks, self.d
        kc, vc = st["kc"], st["vc"]                          # [L][max_len][n][D]
        if pos > 0:
            kc[:, :pos] = torch.stack([s[0] for s in states], dim=2)
            vc[:, :pos] = torch.stack([s[1] for s in states], dim=2)
        anc = self._buf("iface_anc", (n, st["max_len"] + 1), dtype=torch.int32)
        anc.copy_(torch.arange(n, dtype=torch.int32, device=anc.device).view(n, 1).expand_as(anc))   # every slot is its own ancestor
        logp = self.step(st, pos, ys[:, -1].to(torch.int32).contiguous(), anc, n, None)
        new_states = [(kc[:, :ln, b].clone(), vc[:, :ln, b].clone()) for b in range(n)]
        return logp.clone(), new_states

    @torch.no_grad()
    def score(self, ys: torch.Tensor, state, x: torch.Tensor):
        """ScorerInterface.score for one hypothesis (transformer_decoder.py:240-260)."""
        logp, states = self.batch_score(ys.unsqueeze(0), [state], x.unsqueeze(0))
        return logp[0], states[0]

    # ---------------------------------------------------------------- device-side incremental scorer
    @torch.no_grad()
    def init_memory(self, enc_split, U, Tmax, lens32, n_slots, max_len):
        """Project the encoder memory once per utterance (shared by the beam); allocate the self-attention cache."""
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
        st = dict(kvmem=kvmem, U=U, Tmax=Tmax, lens32=lens32, n=n_slots, max_len=max_len,
                  kc=self._buf("kc", (L, max_len, n_slots, D)), vc=self._buf("vc", (L, max_len, n_slots, D)),
                  pe=self._pe(max_len))
        return st

    def _pe(self, length):
        key = ("pe", length)
        if key not in self._ws:
            self._ws[key] = abs_pos_table(length, self.d).to(self.after_norm.weight.device)
        return self._ws[key]

    @torch.no_grad()
    def step(self, st, pos, last_tok, anc, W, step_ptr=None):
        """One decoding position for all n slots: returns log-probabilities [n][V] (buffer reused across steps).
        With ``step_ptr`` (device int32) the position is ``pos + *step_ptr`` so that a captured CUDA graph can be replayed.
        Equivalent of batch_score/forward_one_step (transformer_decoder.py:262-311,191-238)."""
        pk = self._packed
        n, D, H, L, Uu = st["n"], self.d, self.heads, self.num_blocks, self.units
        x = self._buf("x", (n, D))
        xn = self._buf("xn", (2, n, D))
        qkv = self._buf("qkv", (n, 3 * D))
        ctx = self._buf("ctx", (2, n, D))
        q = self._buf("q", (n, D))
        h = self._buf("h", (2, n, Uu))
        call("espb_dec_embed_f32", ptr(last_tok), ptr(pk["emb"]), ptr(st["pe"]), pos, ptr(step_ptr), n, D, math.sqrt(D), ptr(x))
        _count()
        for li, w in enumerate(pk["layers"]):
            layernorm(x, *w["n1"], LN_EPS, out_split=xn)
            linear(xn, w["qkv_w"], qkv, bias=w["qkv_b"])
            call("espb_dec_self_attn_f32", ptr(qkv), ptr(st["kc"][li]), ptr(st["vc"][li]), ptr(anc), anc.shape[1], n, D, H, pos,
                 ptr(step_ptr), st["max_len"], ptr(ctx), n * D)
            _count()
            linear(ctx, w["so_w"], x, bias=w["so_b"], residual=x)
            layernorm(x, *w["n2"], LN_EPS, out_split=xn)
            linear(xn, w["cq_w"], q, bias=w["cq_b"])
            call("espb_dec_src_attn_f32", ptr(q), ptr(st["kvmem"][li, 0]), ptr(st["kvmem"][li, 1]), st["U"], st["Tmax"],
                 ptr(st["lens32"]), W, D, H, ptr(ctx), n * D)
            _count()
            linear(ctx, w["co_w"], x, bias=w["co_b"], residual=x)
            layernorm(x, *w["n3"], LN_EPS, out_split=xn)
            linear(xn, w["w1"], h, bias=w["b1"], act=ACT_RELU, split_out=True)
            linear(h, w["w2"], x, bias=w["b2"], residual=x)
        layernorm(x, *pk["an"], LN_EPS, out_split=xn)
        logp = self._buf("logp", (n, self.odim))
        linear(xn, pk["out_w"], logp, bias=pk["out_b"])
        ops.log_softmax_rows_(logp)
        return logp
