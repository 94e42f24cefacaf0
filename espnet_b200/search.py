"""Utterance-batched, device-resident BatchBeamSearch (joint CTC/attention, attention-only, CTC-only).

Per-utterance results are those of the reference's BatchBeamSearch run on each utterance alone
(espnet2/legacy/nets/batch_beam_search.py, beam_search.py:385-498): same scorer weights
(decoder 1-ctc_weight, ctc ctc_weight, length_bonus `penalty`), pre-beam int(1.5*beam) on the full
scorers, eos handling, maxlen/minlen rules, end detection and final ordering.  What differs is where
the state lives: hypotheses never become Python objects during the search.
"""
from typing import Any, Dict, List, NamedTuple, Union

import torch

from . import ops
from .lib import call, ptr
from .ops import _count


class Hypothesis(NamedTuple):
    """Same fields as espnet2.legacy.nets.beam_search.Hypothesis (beam_search.py:15-31)."""

    yseq: torch.Tensor
    score: Union[float, torch.Tensor] = 0
    scores: Dict[str, Union[float, torch.Tensor]] = dict()
    states: Dict[str, Any] = dict()
    hs: List[torch.Tensor] = []

    def asdict(self) -> dict:
        return self._replace(yseq=self.yseq.tolist(), score=float(self.score),
                             scores={k: float(v) for k, v in self.scores.items()})._asdict()


class BatchBeamSearch(torch.nn.Module):
    """scorers: {"decoder": TransformerDecoder | None, "ctc": CTC | None}; weights as Speech2Text builds them
    (asr_inference.py:310-316).  Zero-weight scorers are dropped (beam_search.py:83-85)."""

    def __init__(self, scorers, weights, beam_size, vocab_size, sos, eos, token_list=None, pre_beam_ratio=1.5,
                 pre_beam_score_key=None, normalize_length=False):
        super().__init__()
        self.weights = dict(weights)
        self.w_dec = float(weights.get("decoder", 0.0)) if scorers.get("decoder") is not None else 0.0
        self.w_ctc = float(weights.get("ctc", 0.0)) if scorers.get("ctc") is not None else 0.0
        self.penalty = float(weights.get("length_bonus", 0.0))
        self.decoder = scorers.get("decoder") if self.w_dec != 0 else None
        self.ctc = scorers.get("ctc") if self.w_ctc != 0 else None
        # LM shallow fusion (asr_inference.py:178-191): a second full scorer with weight lm_weight
        self.w_lm = float(weights.get("lm", 0.0)) if scorers.get("lm") is not None else 0.0
        self.lm = scorers.get("lm") if self.w_lm != 0 else None
        if self.w_lm < 0:
            raise NotImplementedError("negative scorer weights")
        if self.decoder is None and self.ctc is None:
            raise ValueError("no decoder / ctc scorer with non-zero weight")
        if self.decoder is not None and self.w_dec < 0 or self.w_ctc < 0:
            raise NotImplementedError("negative scorer weights")
        self.nn_dict = torch.nn.ModuleDict({k: v for k, v in (("decoder", self.decoder), ("ctc", self.ctc), ("lm", self.lm)) if v is not None})
        self.sos, self.eos, self.n_vocab, self.beam_size = sos, eos, vocab_size, beam_size
        self.token_list = token_list
        self.pre_beam_size = int(pre_beam_ratio * beam_size)
        self.pre_beam_score_key = pre_beam_score_key
        self.do_pre_beam = (pre_beam_score_key is not None and self.pre_beam_size < vocab_size and self.ctc is not None
                            and self.decoder is not None)
        if self.decoder is not None and self.ctc is not None and not self.do_pre_beam:
            raise NotImplementedError("joint decoding without pre-beam (vocab <= 1.5*beam) is not implemented")
        self.normalize_length = normalize_length
        self.full_scorers = {k: v for k, v in (("decoder", self.decoder), ("lm", self.lm)) if v is not None}
        self.part_scorers = {k: v for k, v in (("ctc", self.ctc),) if v is not None}
        if beam_size > 64:
            raise NotImplementedError("beam_size > 64 (beam selection: one block per utterance, 64 slots; cross-attention: groups of 16 slots up to 64)")

    # ---------------------------------------------------------------- search state (cached per shape so that CUDA graphs can be reused)
    def _state(self, dev, U, Tmax, W, V, cap, mode, P, g=0, end_detect=0):
        # end_detect is baked into the captured CUDA graphs (by-value kernel argument of beam_select): it is part of the key
        key = (str(dev), U, Tmax, W, V, cap, mode, P, g, end_detect, self.lm is not None)
        cache = getattr(self, "_state_cache", None)
        if cache is None:
            cache = self._state_cache = {}
        st = cache.get(key)
        if st is not None:
            return st
        if len(cache) >= 8:
            cache.clear()
        n, PC = U * W, (P + 1 if mode == 1 else P)
        i32 = lambda *s: torch.zeros(s, dtype=torch.int32, device=dev)  # noqa: E731
        f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)  # noqa: E731
        ended_cap = W * cap
        st = dict(
            score=[f32(n), f32(n)], sc_dec=[f32(n), f32(n)], sc_ctc=[f32(n), f32(n)], active=[i32(n), i32(n)],
            last_tok=[i32(n), i32(n)], parent=i32(n), anc=[i32(n, cap + 1), i32(n, cap + 1)],
            bp_parent=i32(cap, n), bp_token=i32(cap, n), ended_cap=ended_cap,
            e_count=i32(U), e_step=i32(U, ended_cap), e_slot=i32(U, ended_cap),
            e_score=f32(U, ended_cap), e_dec=f32(U, ended_cap), e_ctc=f32(U, ended_cap),
            best_at=f32(U, cap), best_all=f32(U), done=i32(U), cand_ids=i32(n, P), cand_val=f32(n, P), n_active=i32(1),
            step=i32(1), lens32=i32(U), maxlen=i32(U), minlen=i32(U), graphs={}, graph_launches={})
        if mode != 0:
            st["logp_ctc"] = f32(U * Tmax, V)
            st["r"] = [f32(n, Tmax, 4), f32(n, Tmax, 4)]   # per frame (r^n, r^b, r_sum, pad)
            st["s_prev"] = [f32(n), f32(n)]
            if mode == 1:
                st["part"], st["psi"], st["valid"] = f32(n, PC), f32(n, PC), i32(n, PC)
                st["logp_ctc_t"] = f32(U * V, Tmax)
            else:
                st["part"] = f32(n, V)
        if self.lm is not None:   # second full scorer: combined full scores, per-scorer running scores (ping-pong) and their per-step record
            st["full"] = f32(n, V)
            st["sc_a"], st["sc_b"] = [f32(n), f32(n)], [f32(n), f32(n)]
            st["hist_a"], st["hist_b"] = f32(cap, n), f32(cap, n)
        cache[key] = st
        return st

    use_cuda_graphs = True   # replay one captured graph per step parity once the buffers are warm (steps >= 4)
    # Utterances are independent, and one decoding step is a chain of ~80 small dependent kernels that each fill only part of the GPU:
    # batches of >= group_min_utts utterances are searched as n_groups independent groups on their own streams (own state, decoder
    # workspace and CUDA graphs), stepped in lock-step from the host so that the groups' kernel chains overlap on the device.
    group_min_utts = 16
    n_groups = 1      # one group: the decode-step chains of several groups do not overlap profitably

    def _group_bounds(self, U):
        import os

        G = int(os.environ.get("ESPB_SEARCH_GROUPS", self.n_groups))
        if G <= 1 or U < self.group_min_utts or U < 2 * G:
            return [(0, U)]
        base, rem = divmod(U, G)
        bounds, u0 = [], 0
        for g in range(G):
            u1 = u0 + base + (1 if g < rem else 0)
            bounds.append((u0, u1))
            u0 = u1
        return bounds

    @torch.no_grad()
    def forward_batch(self, enc, enc_lens, enc_split=None, maxlenratio=0.0, minlenratio=0.0, check_every=8):
        """enc (U, Tmax, D) CUDA, enc_lens (U,) -> list (per utterance) of n-best Hypothesis lists, sorted."""
        out = self._search_once(enc, enc_lens, enc_split, maxlenratio, minlenratio, check_every)
        # "there is no N-best results, perform recognition again with smaller minlenratio" (beam_search.py:462-471), per utterance
        empty = [u for u, hyps in enumerate(out) if not hyps]
        if empty and minlenratio >= 0.1:
            idx = torch.tensor(empty, dtype=torch.long, device=enc.device)
            lens_sub = enc_lens.detach().cpu()[torch.tensor(empty)]
            retry = self.forward_batch(enc.index_select(0, idx).contiguous(), lens_sub, None, maxlenratio, max(0.0, minlenratio - 0.1), check_every)
            for u, hyps in zip(empty, retry):
                out[u] = hyps
        return out

    def _search_once(self, enc, enc_lens, enc_split, maxlenratio, minlenratio, check_every):
        U, Tmax, D = enc.shape
        bounds = self._group_bounds(U)
        if len(bounds) == 1:
            run = _SearchRun(self, 0, None, enc, enc_lens, enc_split, maxlenratio, minlenratio)
            self._drive([run], check_every)
            return run.collect()
        main = torch.cuda.current_stream()
        lens_cpu = enc_lens.detach().cpu()
        runs = []
        for g, (u0, u1) in enumerate(bounds):
            sg = self._group_stream(enc.device, g)
            sg.wait_stream(main)
            with torch.cuda.stream(sg):
                es_g = None
                if enc_split is not None:   # hi/lo planes of this group's rows as one contiguous split tensor
                    es_g = enc_split.view(2, U * Tmax, D)[:, u0 * Tmax:u1 * Tmax].contiguous()
                runs.append(_SearchRun(self, g, sg, enc[u0:u1], lens_cpu[u0:u1], es_g, maxlenratio, minlenratio))
        self._drive(runs, check_every)
        out = []
        for r in runs:
            with torch.cuda.stream(r.stream):
                out.extend(r.collect())
            main.wait_stream(r.stream)
        return out

    def _drive(self, runs, check_every):
        """Host loop: step i of every unfinished group is enqueued before any group is polled for termination."""
        import contextlib

        ctx = lambda r: torch.cuda.stream(r.stream) if r.stream is not None else contextlib.nullcontext()  # noqa: E731
        for i in range(max(r.cap for r in runs)):
            live = [r for r in runs if not r.finished and i < r.cap]
            if not live:
                break
            for r in live:
                with ctx(r):
                    r.step(i)
            for r in live:
                if (i + 1) % check_every == 0 or r.end_detect:
                    with ctx(r):
                        r.poll(i)
        for r in runs:
            with ctx(r):
                r.join()

    def _group_stream(self, dev, g):
        key = (str(dev), g)
        if not hasattr(self, "_grp_streams"):
            self._grp_streams = {}
        if key not in self._grp_streams:
            self._grp_streams[key] = torch.cuda.Stream(device=dev)
        return self._grp_streams[key]

    def _capture_stream(self, dev):
        if not hasattr(self, "_cap_streams"):
            self._cap_streams = {}
        key = str(dev)
        if key not in self._cap_streams:
            self._cap_streams[key] = torch.cuda.Stream(device=dev)
        return self._cap_streams[key]

    def _side_stream(self, dev, g=0):
        key = (str(dev), g)
        if not hasattr(self, "_streams"):
            self._streams = {}
        if key not in self._streams:
            self._streams[key] = torch.cuda.Stream(device=dev)
        return self._streams[key]

    def _collect(self, U, W, steps, maxlen, bp_parent, bp_token, e_count, e_step, e_slot, e_score, e_dec, e_ctc, hist=None):
        """Host post-processing: rebuild token sequences from back-pointers and sort (beam_search.py:452-459).
        The back-pointer walk is vectorised over all ended hypotheses (one numpy gather per position)."""
        import numpy as np

        bpp, bpt = bp_parent[:steps].cpu().numpy(), bp_token[:steps].cpu().numpy()
        cnt = e_count.cpu().numpy().astype(np.int64)
        es, el = e_step.cpu().numpy(), e_slot.cpu().numpy()
        sc, sd, sct = e_score.cpu().numpy(), e_dec.cpu().numpy(), e_ctc.cpu().numpy()
        cap_e = es.shape[1]
        sel = np.arange(cap_e)[None, :] < cnt[:, None]                    # [U][cap_e] valid ended entries, utterance-major order
        uu, ee = np.nonzero(sel)
        nh = uu.shape[0]
        step_h, slot_h = es[uu, ee].astype(np.int64), el[uu, ee].astype(np.int64)
        mlen = np.asarray([int(m) for m in maxlen], dtype=np.int64)[uu] if nh else np.zeros(0, np.int64)
        L = int(step_h.max()) + 1 if nh else 0
        # yseq = [sos] + tokens(0..step) (+ eos if the hypothesis was cut at maxlen, batch_beam_search.py:392-407)
        seq = np.full((nh, L + 2), self.eos, dtype=np.int64)
        if nh:
            seq[:, 0] = self.sos
            s = slot_h.copy()
            for j in range(L - 1, -1, -1):
                live = step_h >= j
                sj = s[live]
                seq[live, j + 1] = bpt[j, sj]
                s[live] = bpp[j, sj]
        at_max = step_h == mlen - 1
        length = step_h + 2 + at_max                                      # sos + (step+1) tokens (+ appended eos)
        seq_t = torch.from_numpy(seq)
        score_h, dec_h, ctc_h = sc[uu, ee], sd[uu, ee], sct[uu, ee]
        lm_h = None
        if hist is not None:   # LM fusion: the per-scorer scores were recorded per step (the beam kernel tracked their weighted sum)
            ha, hb = hist[0][:steps].cpu().numpy(), hist[1][:steps].cpu().numpy()
            dec_h, lm_h = (ha[step_h, slot_h], hb[step_h, slot_h]) if nh else (dec_h, np.zeros(0, np.float32))
        key = score_h / (length - 1) if self.normalize_length else score_h
        results = [[] for _ in range(U)]
        start = np.concatenate([[0], np.cumsum(cnt)])
        has_dec, has_ctc, has_pen = self.decoder is not None, self.ctc is not None, self.penalty != 0
        has_lm = lm_h is not None
        for u in range(U):
            lo, hi = int(start[u]), int(start[u + 1])
            if hi == lo:
                continue
            order = lo + np.argsort(-key[lo:hi], kind="stable")         # descending, ties keep ended order (list.sort is stable)
            hyps = results[u]
            for i in order.tolist():
                scores = {}
                if has_dec:
                    scores["decoder"] = float(dec_h[i])
                if has_ctc:
                    scores["ctc"] = float(ctc_h[i])
                if has_lm:
                    scores["lm"] = float(lm_h[i])
                if has_pen:
                    scores["length_bonus"] = float(step_h[i] + 1)
                hyps.append(Hypothesis(yseq=seq_t[i, : int(length[i])], score=float(score_h[i]), scores=scores))
        return results

    def forward(self, x, maxlenratio=0.0, minlenratio=0.0):
        """Reference signature: one utterance, x (T, D) -> n-best list (beam_search.py:385-498)."""
        lens = torch.tensor([x.shape[0]], dtype=torch.int64)
        return self.forward_batch(x.unsqueeze(0).contiguous(), lens, None, maxlenratio, minlenratio)[0]   # incl. the minlenratio retry


class _SearchRun:
    """State and step function of one group of utterances (one stream).  Created by BatchBeamSearch.forward_batch."""

    def __init__(self, bs, g, stream, enc, enc_lens, enc_split, maxlenratio, minlenratio):
        self.bs, self.g, self.stream = bs, g, stream
        dev = enc.device
        U, Tmax, D = enc.shape
        W, V = bs.beam_size, bs.n_vocab
        n = U * W
        lens_cpu = enc_lens.detach().cpu().to(torch.int64)
        if maxlenratio == 0:
            maxlen = lens_cpu.clone()
        elif maxlenratio < 0:
            maxlen = torch.full_like(lens_cpu, -int(maxlenratio))
        else:
            maxlen = torch.clamp((maxlenratio * lens_cpu.double()).long(), min=1)
        minlen = torch.full_like(lens_cpu, -int(minlenratio)) if minlenratio < 0 else (minlenratio * lens_cpu.double()).long()
        cap = int(maxlen.max())
        if enc_split is None:
            enc_split = ops.split_from(enc.contiguous().view(U * Tmax, D))
        use_dec, use_ctc = bs.decoder is not None, bs.ctc is not None
        mode = 1 if (use_dec and use_ctc) else (0 if use_dec else 2)
        P = bs.pre_beam_size if mode == 1 else W
        self.end_detect = 1 if maxlenratio == 0.0 else 0
        st = bs._state(dev, U, Tmax, W, V, cap, mode, P, g, self.end_detect)
        self.U, self.W, self.V, self.n, self.Tmax, self.cap, self.mode, self.P, self.st = U, W, V, n, Tmax, cap, mode, P, st
        self.maxlen, self.use_dec, self.use_ctc, self.dev, self.lens_cpu = maxlen, use_dec, use_ctc, dev, lens_cpu
        self.finished, self.steps_run = False, 0

        # ---- (re)initialise the state in place: one hypothesis [sos] per utterance (batch_beam_search.py:124-153)
        for k in ("score", "sc_dec", "sc_ctc", "active"):
            st[k][0].zero_(); st[k][1].zero_()
        st["active"][0].view(U, W)[:, 0] = 1
        st["last_tok"][0].fill_(bs.sos); st["last_tok"][1].fill_(bs.sos)
        st["bp_parent"].fill_(-1); st["bp_token"].fill_(bs.eos)
        st["e_count"].zero_(); st["done"].zero_()
        st["best_at"].fill_(float("-inf")); st["best_all"].fill_(float("-inf"))
        st["lens32"].copy_(lens_cpu.to(torch.int32)); st["maxlen"].copy_(maxlen.to(torch.int32)); st["minlen"].copy_(minlen.to(torch.int32))
        st["step"].zero_()
        self.lens32 = st["lens32"]
        self.dst = None
        if use_dec:
            bs.decoder.ws_tag = g
            self.dst = bs.decoder.init_memory(enc_split, U, Tmax, self.lens32, n, cap)
        self.lst = None
        if bs.lm is not None:
            bs.lm.ws_tag = g
            self.lst = bs.lm.init_cache(n, cap)
            for k in ("sc_a", "sc_b"):
                st[k][0].zero_(); st[k][1].zero_()
        self.logp_ctc = self.logp_tok = None
        self.tok_major = 0
        if use_ctc:
            self.logp_ctc = bs.ctc.log_softmax(enc, enc_split, out=st["logp_ctc"])   # (U, Tmax, V), scorers/ctc.py:96-99
            call("espb_ctc_init_state_f32", ptr(self.logp_ctc), U, Tmax, V, ptr(self.lens32), 0, W, ptr(st["r"][0]), ptr(st["s_prev"][0]))
            _count()
            self.logp_tok = self.logp_ctc
            if mode == 1:   # token-major copy [U][V][Tmax]: the per-step candidate columns become contiguous reads
                self.logp_tok, self.tok_major = st["logp_ctc_t"], 1
                call("espb_transpose_tv_f32", ptr(self.logp_ctc), U, Tmax, V, ptr(self.logp_tok))
                _count()
        self.side = bs._side_stream(dev, g) if (use_ctc and use_dec) else None
        self.buf_ver = ((getattr(bs.decoder, "buf_version", 0), id(bs.decoder._packed)) if use_dec else None,
                        (getattr(bs.lm, "buf_version", 0), id(bs.lm._packed)) if bs.lm is not None else None)

    def step_body(self, i, cur, sp):
        """One search step. `sp` is None (host step index i) or the device step counter (graph mode: i is ignored)."""
        bs, st = self.bs, self.st
        U, W, V, n, Tmax, P, mode, cap = self.U, self.W, self.V, self.n, self.Tmax, self.P, self.mode, self.cap
        lens32, side = self.lens32, self.side
        score, sc_dec, sc_ctc, active, last_tok = st["score"], st["sc_dec"], st["sc_ctc"], st["active"], st["last_tok"]
        parent, anc = st["parent"], st["anc"]
        r, s_prev = st.get("r"), st.get("s_prev")
        nxt = cur ^ 1
        iv = 0 if sp is not None else i
        main = torch.cuda.current_stream()
        forked = False
        if self.use_ctc and (sp is not None or i >= 1):
            # CTC forward variables of the hypotheses chosen in the previous step (scorers/ctc.py:40-63): only the scoring below needs
            # them, so the T-step recursion runs on a side stream concurrently with the decoder pass
            def advance():
                call("espb_ctc_advance_f32", ptr(self.logp_tok), U, Tmax, V, ptr(lens32), 0, bs.eos, W, ptr(r[nxt]), ptr(parent),
                     ptr(last_tok[nxt]), ptr(last_tok[cur]), ptr(active[cur]), iv - 1, ptr(sp), ptr(r[cur]), ptr(s_prev[cur]), self.tok_major)
                _count()
            if side is not None:
                ev = torch.cuda.Event()
                ev.record(main)
                with torch.cuda.stream(side):
                    side.wait_event(ev)
                    advance()
                forked = True
            else:
                advance()
        logp_dec = None
        if self.use_dec:
            bs.decoder.ws_tag = self.g
            logp_dec = bs.decoder.step(self.dst, iv, last_tok[cur], anc[cur], W, sp)
        logp_lm, w_full, logp_full = None, bs.w_dec, logp_dec
        if bs.lm is not None:
            bs.lm.ws_tag = self.g
            logp_lm = bs.lm.step(self.lst, iv, last_tok[cur], anc[cur], sp)
            if self.use_dec:   # weighted sum of the full scorers, decoder first (batch_beam_search.py:293-300); the beam kernels then see one scorer of weight 1
                call("espb_axpby_f32", ptr(logp_dec), bs.w_dec, ptr(logp_lm), bs.w_lm, ptr(st["full"]), n * V)
                _count()
                w_full, logp_full = 1.0, st["full"]
        if forked:
            main.wait_stream(side)
        if mode == 1:
            ops.rows_topk(logp_full, w_full, P, st["cand_ids"], st["cand_val"])
            call("espb_ctc_score_cands_f32", ptr(self.logp_tok), U, Tmax, V, ptr(lens32), 0, bs.eos, W, ptr(r[cur]), ptr(s_prev[cur]),
                 ptr(last_tok[cur]), iv, ptr(sp), ptr(st["cand_ids"]), P, ptr(st["part"]), ptr(st["psi"]), ptr(st["valid"]), self.tok_major)
            _count()
        elif mode == 0:
            ops.rows_topk(logp_full, w_full, P, st["cand_ids"], st["cand_val"])
        else:
            call("espb_ctc_score_dense_f32", ptr(self.logp_ctc), U, Tmax, V, ptr(lens32), 0, bs.eos, W, ptr(r[cur]), ptr(s_prev[cur]),
                 ptr(last_tok[cur]), i, ptr(st["part"]))
            _count()
            if logp_lm is not None:   # CTC-only + LM: the LM is the only full scorer, no pre-beam: (w_lm * lm) + (w_ctc * ctc) over the vocabulary
                call("espb_axpby_f32", ptr(logp_lm), bs.w_lm, ptr(st["part"]), bs.w_ctc, ptr(st["full"]), n * V)
                _count()
                ops.rows_topk(st["full"], 1.0, P, st["cand_ids"], st["cand_val"])
            else:
                ops.rows_topk(st["part"], bs.w_ctc, P, st["cand_ids"], st["cand_val"])
        call("espb_beam_select", ptr(score[cur]), ptr(sc_dec[cur]), ptr(sc_ctc[cur]), ptr(active[cur]), ptr(score[nxt]),
             ptr(sc_dec[nxt]), ptr(sc_ctc[nxt]), ptr(active[nxt]), ptr(last_tok[nxt]), ptr(parent), ptr(st["bp_parent"]),
             ptr(st["bp_token"]), ptr(st["e_count"]), ptr(st["e_step"]), ptr(st["e_slot"]), ptr(st["e_score"]), ptr(st["e_dec"]),
             ptr(st["e_ctc"]), st["ended_cap"], ptr(st["best_at"]), ptr(st["best_all"]), ptr(st["done"]), U, W, P, V, iv, ptr(sp),
             ptr(st["maxlen"]), ptr(st["minlen"]), bs.eos, w_full, bs.w_ctc, bs.penalty, mode, ptr(st["cand_ids"]),
             ptr(st["cand_val"]), ptr(logp_full), ptr(st.get("part")), ptr(st.get("valid")), self.end_detect, cap)
        _count()
        if logp_lm is not None:   # per-scorer scores of the chosen hypotheses (the beam kernel only tracked the combined full score)
            call("espb_track_scores_f32", ptr(parent), ptr(last_tok[nxt]), ptr(st["bp_parent"]), ptr(logp_dec), ptr(logp_lm), V, ptr(st["sc_a"][cur]),
                 ptr(st["sc_b"][cur]), ptr(st["sc_a"][nxt]), ptr(st["sc_b"][nxt]), ptr(st["hist_a"]), ptr(st["hist_b"]), iv, ptr(sp), n)
            _count()
        if self.use_dec or logp_lm is not None:
            call("espb_anc_update_i32", ptr(anc[cur]), ptr(anc[nxt]), cap + 1, ptr(parent), iv, ptr(sp), n)
            _count()
        if sp is not None:
            call("espb_step_inc_i32", ptr(sp))
            _count()

    def step(self, i):
        from . import lib as _lib

        bs, st = self.bs, self.st
        step_dev = st["step"]
        graphs_ok = (bs.use_cuda_graphs and self.mode != 2 and self.cap >= 8 and _lib.profile is None and ops.gemm_profile is None)
        cur = i & 1
        if graphs_ok and i >= 2:
            if st.get("graph_buf_ver") != self.buf_ver:   # decoder buffers / packed weights were re-created: captured pointers are stale
                st["graphs"].clear()
                st["graph_buf_ver"] = self.buf_ver
            g = st["graphs"].get(cur)
            if g is None:      # capture this parity once (steps 2 and 3); nothing executes during capture, so replay right after
                step_dev.fill_(i)
                g = torch.cuda.CUDAGraph()
                cs = bs._capture_stream(self.dev)
                cs.wait_stream(torch.cuda.current_stream())
                before = ops.launch_counter[0]
                with torch.cuda.stream(cs):
                    g.capture_begin()
                    self.step_body(i, cur, step_dev)
                    g.capture_end()
                torch.cuda.current_stream().wait_stream(cs)
                st["graph_launches"][cur] = ops.launch_counter[0] - before
                ops.launch_counter[0] = before
                st["graphs"][cur] = g
            elif i == 2:
                step_dev.fill_(i)  # graphs cached from an earlier call: (re)position the device step counter
            g.replay()
            ops.launch_counter[0] += st["graph_launches"][cur]
        else:
            self.step_body(i, cur, None)
        self.steps_run = i + 1

    def poll(self, i):
        st = self.st
        call("espb_count_active_i32", ptr(st["active"][(i + 1) & 1]), self.n, ptr(st["n_active"]))
        _count()
        if int(st["n_active"].item()) == 0:
            self.finished = True

    def join(self):
        if self.side is not None:
            torch.cuda.current_stream().wait_stream(self.side)

    def collect(self):
        st = self.st
        if self.use_ctc:
            # The prefix scorer indexes its forward variables at [len(prefix) - 1] (ctc_prefix_score.py:147-172): the reference raises an
            # IndexError in the middle of decoding once a LIVE hypothesis is two tokens longer than the encoder output.  The kernels keep an
            # all-logzero state there instead of indexing out of bounds; an utterance is reported only if that really happened, i.e. a
            # hypothesis of it was still being extended at step T + 1 (back-pointer rows of dead slots are -1).
            over = [u for u in range(self.U) if int(self.maxlen[u]) > int(self.lens_cpu[u]) + 1 and self.steps_run > int(self.lens_cpu[u]) + 1]
            if over:
                bpp = st["bp_parent"][: self.steps_run].cpu()
                bad = [u for u in over if bool((bpp[int(self.lens_cpu[u]) + 1, u * self.W:(u + 1) * self.W] >= 0).any())]
                if bad:
                    u = bad[0]
                    raise IndexError(f"CTC prefix scoring cannot extend hypotheses beyond the encoder output length + 1: utterance(s) {bad} of this group "
                                     f"still had live hypotheses at step {int(self.lens_cpu[u]) + 1} ({int(self.lens_cpu[u])} encoder frames, maxlen "
                                     f"{int(self.maxlen[u])}); lower maxlenratio or decode with ctc_weight=0")
        hist = (st["hist_a"], st["hist_b"]) if self.bs.lm is not None else None
        return self.bs._collect(self.U, self.W, self.steps_run, self.maxlen, st["bp_parent"], st["bp_token"], st["e_count"], st["e_step"],
                                st["e_slot"], st["e_score"], st["e_dec"], st["e_ctc"], hist)
