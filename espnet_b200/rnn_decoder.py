"""RNNDecoder (LSTM decoder with location-aware attention) with the reference's constructor / state_dict surface, as a device-side
incremental scorer of the beam search.

Reference: espnet2/asr/decoder/rnn_decoder.py (RNNDecoder: init_state / score), legacy/nets/pytorch_backend/rnn/attentions.py:249-378
(AttLoc).  One step for the n hypothesis slots:
  1. one gather: the embedding of the newest token and every layer's parent h into the gate GEMM operands (espb_rnnlm_gather_f32, shared
     with the LSTM LM);
  2. mlp_dec over the parent's first-layer h (a GEMM reading the recurrent half of layer 0's operand);
  3. the attention step (espb_att_loc_step_f32): location conv over the parent's previous weights, mlp_att, energies against the
     per-utterance mlp_enc(enc) computed once in init_memory, masked softmax(2 e), new weights into the ring, context into the operands;
  4. per layer one GEMM [input | parent h] @ [W_ih | W_hh]^T + b and one cell kernel (espb_lstm_cell_f32), then the output GEMM
     (on [z_L | c] with context_residual) and log-softmax.
The recurrent state h, c [2][L][n][Hp] and the previous attention weights [2][n][Tmax] are two-deep rings addressed through the search's
ancestor table, as SequentialRNNLM's h / c: nothing is copied when the beam is reordered.  Layer 0's operand is [embed | c | parent h],
each part padded to a multiple of 4 columns (TMA strides) with zero columns in weights and operands.

The reference decodes this model with its non-batch BeamSearch (RNNDecoder is a ScorerInterface, not a BatchScorerInterface); ``score``
implements that protocol on the same kernels.
"""
from typing import Any, Tuple

import torch

from . import ops
from .layers import PackedModule
from .lib import call, ptr
from .ops import _count, linear, split_from


def _pad4(k):
    return (k + 3) & ~3


class _AttLoc(torch.nn.Module):
    def __init__(self, eprojs, dunits, att_dim, aconv_chans, aconv_filts):
        super().__init__()
        self.mlp_enc = torch.nn.Linear(eprojs, att_dim)
        self.mlp_dec = torch.nn.Linear(dunits, att_dim, bias=False)
        self.mlp_att = torch.nn.Linear(aconv_chans, att_dim, bias=False)
        self.loc_conv = torch.nn.Conv2d(1, aconv_chans, (1, 2 * aconv_filts + 1), padding=(0, aconv_filts), bias=False)
        self.gvec = torch.nn.Linear(att_dim, 1)


class RNNDecoder(PackedModule):
    """Drop-in container for espnet2.asr.decoder.rnn_decoder.RNNDecoder (inference scorer): LSTM cells, one encoder, ``atype: location``."""

    zero_bufs = True   # the operands' pad columns are zeroed when the buffers are created and never written afterwards
    # RNNDecoder is a non-batch ScorerInterface, so the reference decodes it with BeamSearch, in which <eos> is a candidate only when the
    # pre-beam of the full scores holds it (espnet_b200.BatchBeamSearch follows that rule for this decoder)
    eos_from_prebeam_only = True

    def __init__(self, vocab_size: int, encoder_output_size: int, rnn_type: str = "lstm", num_layers: int = 1, hidden_size: int = 320,
                 sampling_probability: float = 0.0, dropout: float = 0.0, context_residual: bool = False, replace_sos: bool = False,
                 num_encs: int = 1, att_conf: dict = None):
        super().__init__()
        if rnn_type not in {"lstm", "gru"}:
            raise ValueError(f"Not supported: rnn_type={rnn_type}")
        att = dict(atype="location", num_att=1, num_encs=1, aheads=4, adim=320, awin=5, aconv_chans=10, aconv_filts=100, han_mode=False,
                   han_type=None, han_heads=4, han_dim=320, han_conv_chans=-1, han_conv_filts=100, han_win=5)
        unknown = set(att_conf or {}) - set(att)
        if unknown:
            raise TypeError(f"build_attention_list() got unexpected keyword arguments {sorted(unknown)}")
        han_defaults = {k: att[k] for k in att if k.startswith("han_")}
        att.update(att_conf or {})
        unsupported = []
        if rnn_type == "gru": unsupported.append("rnn_type=gru")
        if att["atype"] != "location": unsupported.append(f"atype={att['atype']}")
        if num_encs != 1 or att["num_encs"] != 1: unsupported.append("num_encs > 1")
        if att["num_att"] != 1: unsupported.append(f"num_att={att['num_att']}")
        if replace_sos: unsupported.append("replace_sos")
        if sampling_probability > 0: unsupported.append("sampling_probability > 0")
        if any(att[k] != v for k, v in han_defaults.items()): unsupported.append("han_* options")
        if unsupported:
            raise NotImplementedError("espnet_b200.RNNDecoder does not implement: " + ", ".join(unsupported))
        H, E = hidden_size, encoder_output_size
        self.dunits, self.dlayers, self.eprojs, self.odim = H, num_layers, E, vocab_size
        self.context_residual = context_residual
        self.sos = self.eos = vocab_size - 1
        self.adim, self.aconv_chans, self.aconv_filts = att["adim"], att["aconv_chans"], att["aconv_filts"]
        self.embed = torch.nn.Embedding(vocab_size, H)
        self.decoder = torch.nn.ModuleList([torch.nn.LSTMCell(H + E, H)] + [torch.nn.LSTMCell(H, H) for _ in range(1, num_layers)])
        self.output = torch.nn.Linear(H + E if context_residual else H, vocab_size)
        self.att_list = torch.nn.ModuleList([_AttLoc(E, H, self.adim, self.aconv_chans, self.aconv_filts)])

    # ---------------------------------------------------------------- packing
    def _widths(self):
        """(Hp, Cp, Ep, xo width): hidden and context widths padded to 4, layer 0's input half [embed | c] and the output operand."""
        Hp, Cp = _pad4(self.dunits), _pad4(self.eprojs)
        return Hp, Cp, Hp + Cp, Hp + (Cp if self.context_residual else 0)

    def _pack(self):
        f32, dev = self._f32, self._device
        H, E, V, A = self.dunits, self.eprojs, self.odim, self.adim
        Hp, Cp, Ep, Wo = self._widths()
        pk = dict(emb=f32(self.embed.weight), layers=[])
        for k, cell in enumerate(self.decoder):
            ip = Ep if k == 0 else Hp
            w = torch.zeros(4 * H, ip + Hp, dtype=torch.float32, device=dev)
            wih = f32(cell.weight_ih)
            if k == 0:   # input [embed(y); c]
                w[:, :H], w[:, Hp:Hp + E] = wih[:, :H], wih[:, H:]
            else:
                w[:, :H] = wih
            w[:, ip:ip + H] = f32(cell.weight_hh)
            pk["layers"].append((split_from(w), f32(cell.bias_ih) + f32(cell.bias_hh)))
        wo = torch.zeros(V, Wo, dtype=torch.float32, device=dev)
        wo[:, :H] = f32(self.output.weight)[:, :H]
        if self.context_residual:
            wo[:, Hp:Hp + E] = f32(self.output.weight)[:, H:]
        pk["out_w"], pk["out_b"] = split_from(wo), f32(self.output.bias)
        a = self.att_list[0]
        wd = torch.zeros(A, Hp, dtype=torch.float32, device=dev)
        wd[:, :H] = f32(a.mlp_dec.weight)
        pk.update(enc_w=split_from(f32(a.mlp_enc.weight)), enc_b=f32(a.mlp_enc.bias), dec_w=split_from(wd),
                  conv_w=f32(a.loc_conv.weight).view(self.aconv_chans, -1).contiguous(), att_wt=f32(a.mlp_att.weight).t().contiguous(),
                  gvec=f32(a.gvec.weight).view(-1).contiguous(), gvec_b=f32(a.gvec.bias))
        self._packed = pk
        return pk

    # ---------------------------------------------------------------- device-side incremental scorer
    @torch.no_grad()
    def init_memory(self, enc_split, U, Tmax, lens32, n_slots, max_len):
        """mlp_enc of the encoder output once per utterance (shared by its beam) and the state rings of n_slots hypotheses; slot s belongs to
        utterance s // (n_slots / U).  enc_split: split [2][U*Tmax][eprojs]; the rings do not depend on max_len."""
        pk = self._packed or self._pack()
        E, A, L = self.eprojs, self.adim, self.dlayers
        Hp = _pad4(self.dunits)
        M = U * Tmax
        enc_h = self._buf("enc_h", (M, A))
        ops.gemm(M, A, E, enc_split, M * E, E, pk["enc_w"], A * E, E, enc_h, A, bias=pk["enc_b"])
        return dict(n=n_slots, U=U, W=n_slots // U, Tmax=Tmax, lens32=lens32, enc_split=enc_split, enc_h=enc_h,
                    h=self._buf("h", (2, L, n_slots, Hp)), c=self._buf("c", (2, L, n_slots, Hp)), a=self._buf("a", (2, n_slots, Tmax)))

    @torch.no_grad()
    def step(self, st, pos, last_tok, anc, step_ptr=None):
        """One position for all n slots: log-probabilities [n][V] of the next token (buffer reused across steps).  Equivalent of score
        (rnn_decoder.py) for hypotheses whose newest token is ``last_tok`` at position ``pos`` (+ *step_ptr) and whose parent state is ring
        (pos-1)&1 at slot anc[s][pos-1]."""
        pk = self._packed
        n, L, H, E, A = st["n"], self.dlayers, self.dunits, self.eprojs, self.adim
        Hp, Cp, Ep, Wo = self._widths()
        kp0, kp1 = Ep + Hp, 2 * Hp
        xs = self._buf("xs", (2 * n * kp0 + 2 * (L - 1) * n * kp1,))
        xo = self._buf("xo", (2, n, Wo))
        gates = self._buf("gates", (n, 4 * H))
        dec_z = self._buf("dec_z", (n, A))
        ops_ = [xs[:2 * n * kp0].view(2, n, kp0)] + [xs[2 * n * kp0 + 2 * l * n * kp1:2 * n * kp0 + 2 * (l + 1) * n * kp1].view(2, n, kp1)
                                                       for l in range(L - 1)]
        x0 = ops_[0]
        call("espb_rnnlm_gather_f32", ptr(last_tok), ptr(pk["emb"]), H, Ep, ptr(anc), anc.shape[1], pos, ptr(step_ptr), ptr(st["h"]), L, n, H, Hp,
             ptr(xs))
        _count()
        # dec_z = mlp_dec(z_prev[0]): the parent's first-layer h is the recurrent half of layer 0's operand
        ops.gemm(n, A, Hp, x0, n * kp0, kp0, pk["dec_w"], A * Hp, Hp, dec_z, A, a_off=Ep)
        call("espb_att_loc_step_f32", ptr(st["enc_h"]), ptr(st["enc_split"]), st["enc_split"][0].numel(), ptr(st["lens32"]), st["W"], st["Tmax"],
             A, E, ptr(dec_z), ptr(pk["conv_w"]), self.aconv_chans, self.aconv_filts, ptr(pk["att_wt"]), ptr(pk["gvec"]), ptr(pk["gvec_b"]),
             ptr(anc), anc.shape[1], pos, ptr(step_ptr), ptr(st["a"]), n, ptr(x0[0, 0, Hp:]), n * kp0, kp0,
             ptr(xo[0, 0, Hp:]) if self.context_residual else None, n * Wo, Wo)
        _count()
        for li, (w, b) in enumerate(pk["layers"]):
            linear(ops_[li], w, gates, bias=b)
            nxt = ops_[li + 1] if li + 1 < L else xo
            call("espb_lstm_cell_f32", ptr(gates), ptr(anc), anc.shape[1], pos, ptr(step_ptr), ptr(st["h"]), ptr(st["c"]), li, L, n, H, Hp,
                 ptr(nxt), nxt[0].numel(), nxt.shape[2])
            _count()
        logp = self._buf("logp", (n, self.odim))
        linear(xo, pk["out_w"], logp, bias=pk["out_b"])
        ops.log_softmax_rows_(logp)
        return logp

    # ---------------------------------------------------------------- ScorerInterface (legacy/nets/scorer_interface.py), non-batch
    def init_state(self, x: torch.Tensor):
        """Zero h / c and uniform attention weights, represented by None (rnn_decoder.py init_state)."""
        return None

    def select_state(self, state, i: int, new_id: int = None):
        return state

    def final_score(self, state) -> float:
        return 0.0

    def _iface_state(self, x):
        """State for one hypothesis over the encoder output x (T, eprojs): mlp_enc computed once and kept while x is the same tensor."""
        key = (x.data_ptr(), tuple(x.shape), tuple(x.stride()), x._version)
        c = getattr(self, "_iface", None)
        if c is None or c["key"] != key or self._packed is None:
            T = x.shape[0]
            self.ws_tag = "iface"
            # x_ref keeps the storage alive, so that an equal key means the same data
            c = self._iface = dict(key=key, x_ref=x, enc_split=split_from(x.contiguous().float()))
            c["st"] = self.init_memory(c["enc_split"], 1, T, torch.tensor([T], dtype=torch.int32, device=x.device), 1, 1)
        return c["st"]

    @torch.no_grad()
    def score(self, yseq: torch.Tensor, state: Any, x: torch.Tensor) -> Tuple[torch.Tensor, Any]:
        """rnn_decoder.py score: yseq (len,) int64 prefix, state None or (h [L][H], c [L][H], previous attention weights [T]), x (T, eprojs)
        -> (log-probabilities (V,), new state)."""
        self.ws_tag = "iface"
        st = self._iface_state(x)
        H = self.dunits
        pos = 0 if state is None else 1
        if pos:     # parent in ring 0, slot 0
            st["h"][0, :, 0, :H] = state[0]
            st["c"][0, :, 0, :H] = state[1]
            st["a"][0, 0] = state[2]
        anc = self._buf("iface_anc", (1, 1), dtype=torch.int32)
        anc.zero_()
        logp = self.step(st, pos, yseq[-1:].to(torch.int32).contiguous(), anc, None)
        r = pos & 1
        return logp[0].clone(), (st["h"][r, :, 0, :H].clone(), st["c"][r, :, 0, :H].clone(), st["a"][r, 0].clone())
