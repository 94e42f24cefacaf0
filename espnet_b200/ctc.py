"""CTC head (espnet2/asr/ctc.py:13-215): ``ctc_lo`` Linear + log_softmax / argmax, plus on-device greedy collapse."""
import torch

from . import ops
from .layers import PackedModule
from .lib import call, ptr
from .ops import _count, linear, split_from


class CTC(PackedModule):
    def __init__(self, odim: int, encoder_output_size: int, dropout_rate: float = 0.0, ctc_type: str = "builtin",
                 reduce: bool = True, ignore_nan_grad=None, zero_infinity: bool = True, brctc_risk_strategy: str = "exp",
                 brctc_group_strategy: str = "end", brctc_risk_factor: float = 0.0):
        super().__init__()
        self.ctc_lo = torch.nn.Linear(encoder_output_size, odim)
        self.odim, self.eprojs = odim, encoder_output_size

    def _pack(self):
        self._packed = (split_from(self._f32(self.ctc_lo.weight)), self._f32(self.ctc_lo.bias))
        return self._packed

    def _split_input(self, hs_pad, hs_split):
        if hs_split is not None:
            return hs_split
        return split_from(hs_pad.contiguous().float().view(-1, hs_pad.shape[-1]))

    @torch.no_grad()
    def logits(self, hs_pad, hs_split=None, out=None):
        """(B, T, D) -> (B, T, V) = ctc_lo(hs_pad); `out` optionally provides the (B*T, V) result buffer."""
        w, b = self._packed or self._pack()
        B, T, D = hs_pad.shape
        xs = self._split_input(hs_pad, hs_split)
        if out is None:
            out = torch.empty(B * T, self.odim, dtype=torch.float32, device=hs_pad.device)
        out = out.view(B * T, self.odim)
        linear(xs, w, out, bias=b)
        return out.view(B, T, self.odim)

    @torch.no_grad()
    def log_softmax(self, hs_pad, hs_split=None, out=None):
        lg = self.logits(hs_pad, hs_split, out)
        ops.log_softmax_rows_(lg.view(-1, self.odim))
        return lg

    @torch.no_grad()
    def argmax(self, hs_pad, hs_split=None):
        lg = self.logits(hs_pad, hs_split)
        out = torch.empty(lg.shape[0] * lg.shape[1], dtype=torch.int32, device=lg.device)
        ops.argmax_rows(lg.view(-1, self.odim), out)
        return out.view(lg.shape[0], lg.shape[1]).long()

    @torch.no_grad()
    def greedy(self, hs_pad, hlens, hs_split=None, blank=0):
        """argmax -> unique_consecutive -> drop blank, on device.  Returns (ids (B, T) int32, counts (B,) int32, argmax (B,T) int32)."""
        lg = self.logits(hs_pad, hs_split)
        B, T, V = lg.shape
        am = torch.empty(B, T, dtype=torch.int32, device=lg.device)
        ops.argmax_rows(lg.view(-1, V), am)
        ids = torch.zeros(B, T, dtype=torch.int32, device=lg.device)
        cnt = torch.zeros(B, dtype=torch.int32, device=lg.device)
        lens32 = hlens.to(device=lg.device, dtype=torch.int32).contiguous()
        call("espb_ctc_collapse_i32", ptr(am), B, T, ptr(lens32), blank, ptr(ids), ptr(cnt))
        _count()
        return ids, cnt, am


LOGZERO = -10000000000.0


class _CTCHypState:
    """CTC forward variables of one hypothesis: r [T][4] = (r^n, r^b, logaddexp(r^n, r^b), 0) per frame, s = log psi of its prefix."""

    __slots__ = ("r", "s")

    def __init__(self, r, s):
        self.r, self.s = r, s


class _CTCBatchState:
    """What batch_score_partial hands back to the search: the scored hypotheses' previous states; select_state advances one of them."""

    __slots__ = ("r_prev", "last_tok", "out_len")

    def __init__(self, r_prev, last_tok, out_len):
        self.r_prev, self.last_tok, self.out_len = r_prev, last_tok, out_len


class CTCPrefixScorer:
    """BatchPartialScorerInterface over the CUDA CTC prefix-scoring kernels, so that the reference's own BatchBeamSearch can use them
    (espnet2/legacy/nets/scorers/ctc.py:10-157 over ctc_prefix_score.py:71-224; protocol: scorer_interface.py:85-188).

    batch_init_state(x) computes the CTC posteriors of the utterance once (as scorers/ctc.py:96-99); batch_score_partial returns
    ``log_psi - s_prev`` scattered into (n, V) (-1e10 - s_prev for unscored tokens, the eos column always scored, blank = -1e10) exactly like
    CTCPrefixScoreTH.__call__; select_state(state, i, new_id) runs the T-step forward recursion for the chosen (hypothesis, token) only
    (the reference computes it for all n x k candidates and indexes).  espnet_b200.BatchBeamSearch does not go through this class."""

    def __init__(self, ctc: CTC, eos: int):
        self.ctc, self.eos, self.blank = ctc, eos, 0
        self.logp = self.logp_tok = self.lens32 = None

    # -- protocol
    def init_state(self, x: torch.Tensor):
        return self.batch_init_state(x)

    @torch.no_grad()
    def batch_init_state(self, x: torch.Tensor):
        T, V = x.shape[0], self.ctc.odim
        self.T, self.V = T, V
        self.logp = self.ctc.log_softmax(x.unsqueeze(0).contiguous().float()).view(T, V).contiguous()
        self.logp_tok = torch.empty(V, T, dtype=torch.float32, device=x.device)
        call("espb_transpose_tv_f32", ptr(self.logp), 1, T, V, ptr(self.logp_tok))
        self.lens32 = torch.tensor([T], dtype=torch.int32, device=x.device)
        self.r0 = torch.empty(1, T, 4, dtype=torch.float32, device=x.device)
        s0 = torch.empty(1, dtype=torch.float32, device=x.device)
        call("espb_ctc_init_state_f32", ptr(self.logp), 1, T, V, ptr(self.lens32), self.blank, 1, ptr(self.r0), ptr(s0))
        _count(2)
        return None

    def final_score(self, state) -> float:
        return 0.0

    # -- streaming extension (scorers/ctc.py:128-157 over ctc_prefix_score.py:226-270; Eq. 14 of arXiv:2006.14941)
    @torch.no_grad()
    def extend_prob(self, x: torch.Tensor):
        """x (T_new, D): the encoder output so far, grown by a block.  The posteriors are per frame, so recomputing all of them equals the
        reference's 'keep the old rows, append the new ones'."""
        if self.logp is None or x.shape[0] > self.T:
            self.batch_init_state(x)

    @torch.no_grad()
    def extend_state(self, state):
        """List of per-hypothesis states (None before the first step) -> states over the extended posteriors."""
        todo = [i for i, st in enumerate(state) if st is not None and st.r.shape[0] < self.T]
        if not todo:
            return list(state)
        out = list(state)
        by_len = {}
        for i in todo:
            by_len.setdefault(state[i].r.shape[0], []).append(i)
        for t_old, idx in by_len.items():
            r_old = torch.stack([state[i].r for i in idx]).contiguous()
            r_new = torch.empty(len(idx), self.T, 4, dtype=torch.float32, device=r_old.device)
            call("espb_ctc_extend_state_f32", ptr(self.logp), self.T, self.V, self.blank, len(idx), ptr(r_old), t_old, ptr(r_new))
            _count()
            for j, i in enumerate(idx):
                out[i] = _CTCHypState(r_new[j], state[i].s)
        return out

    @torch.no_grad()
    def batch_score_partial(self, y: torch.Tensor, ids: torch.Tensor, state, x: torch.Tensor):
        """y (n, len) int64 prefixes, ids (n, k) int64 tokens to score, state: list of n hypothesis states (None before the first step)."""
        n = y.shape[0]
        dev = y.device
        out_len = y.shape[1] - 1
        if state is None or state[0] is None:
            r_prev = self.r0.expand(n, self.T, 4).contiguous()
            s_prev = torch.zeros(n, dtype=torch.float32, device=dev)
        else:
            r_prev = torch.stack([s.r for s in state]).contiguous()
            s_prev = torch.stack([s.s for s in state]).contiguous()
        last_tok = y[:, -1].to(torch.int32).contiguous()
        if ids is None:     # no pre-beam (CTC-only decoding): every token is scored (ctc_prefix_score.py:118-122)
            scores = torch.empty(n, self.V, dtype=torch.float32, device=dev)
            call("espb_ctc_score_dense_f32", ptr(self.logp), 1, self.T, self.V, ptr(self.lens32), self.blank, self.eos, n, ptr(r_prev), ptr(s_prev),
                 ptr(last_tok), out_len, ptr(scores))
            _count()
            return scores, _CTCBatchState(r_prev, last_tok, out_len)
        k = ids.shape[1]
        cand = ids.to(torch.int32).contiguous()
        part = torch.empty(n, k + 1, dtype=torch.float32, device=dev)
        psi = torch.empty(n, k + 1, dtype=torch.float32, device=dev)
        valid = torch.empty(n, k + 1, dtype=torch.int32, device=dev)
        call("espb_ctc_score_cands_f32", ptr(self.logp_tok), 1, self.T, self.V, ptr(self.lens32), self.blank, self.eos, n, ptr(r_prev), ptr(s_prev),
             ptr(last_tok), out_len, None, ptr(cand), k, ptr(part), ptr(psi), ptr(valid), 1)
        _count()
        scores = (LOGZERO - s_prev).unsqueeze(1).repeat(1, self.V)
        scores.scatter_(1, ids.long(), part[:, :k])
        scores[:, self.eos] = part[:, k]                      # the eos column is always scored (ctc_prefix_score.py:184-185)
        if self.eos != self.blank:
            scores[:, self.blank] = LOGZERO - s_prev          # (:187-189)
        return scores, _CTCBatchState(r_prev, last_tok, out_len)

    @torch.no_grad()
    def select_state(self, state, i, new_id=None):
        if state is None:
            return None
        if isinstance(state, (list, tuple)):
            return state[i]
        if isinstance(state, _CTCHypState):
            return state
        dev = state.r_prev.device
        i, tok = int(i), int(new_id)
        parent = torch.tensor([i], dtype=torch.int32, device=dev)
        new_tok = torch.tensor([tok], dtype=torch.int32, device=dev)
        active = torch.ones(1, dtype=torch.int32, device=dev)
        r_new = torch.empty(1, self.T, 4, dtype=torch.float32, device=dev)
        s_new = torch.empty(1, dtype=torch.float32, device=dev)
        call("espb_ctc_advance_f32", ptr(self.logp_tok), 1, self.T, self.V, ptr(self.lens32), self.blank, self.eos, 1, ptr(state.r_prev), ptr(parent),
             ptr(state.last_tok), ptr(new_tok), ptr(active), state.out_len, None, ptr(r_new), ptr(s_new), 1)
        _count()
        return _CTCHypState(r_new[0], s_new[0])

    def score_partial(self, y, next_tokens, state, x):
        raise NotImplementedError("espnet_b200.CTCPrefixScorer implements the batch protocol (batch_score_partial): use BatchBeamSearch")
