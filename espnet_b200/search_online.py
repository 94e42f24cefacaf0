"""Block-synchronous beam search for streaming decoding (SURVEY.md 8f-2; Tsunoo et al., arXiv:2006.14941).

Reference: espnet2/legacy/nets/batch_beam_search_online.py:22-534 (``BatchBeamSearchOnline``: block-wise processing with rewinding) over
batch_beam_search.py:253-423 (one search step, post-processing) and beam_search.py:66-113 (scorer / pre-beam configuration).  One instance decodes
one live stream: every push appends encoder frames to the stream's buffer; for every block boundary the buffer now covers the search runs over the
frames up to that boundary until a hypothesis reaches <eos> or repeats a token -- both mean "the decoder has run past the audio it has seen" -- then
rewinds one step and waits for the next block.

The scorers are the CUDA-backed protocol classes of this package (``TransformerDecoder.batch_score``, ``CTCPrefixScorer.batch_score_partial`` with
``extend_prob`` / ``extend_state`` for the growing encoder output, ``TransformerLM.batch_score``, ``LengthBonus``): the same scorer protocol as the
reference (scorer_interface.py:85-188), so the running set lives in a handful of device tensors (token matrix, total and per-scorer scores) plus one
state list per scorer, instead of a Python object per hypothesis.

Not implemented (refused): time-synchronous / transducer streaming search, ``block_size == 0`` (recompute mode), ``encoded_feat_length_limit`` and
``decoder_text_length_limit``.
"""
import logging
import math
from typing import Any, Dict, List, Optional

import torch

from .decoder import ScorerProtocol
from .search import Hypothesis


class LengthBonus(ScorerProtocol):
    """Constant 1 per emitted token (espnet2/legacy/nets/scorers/length_bonus.py:10-62): weight ``penalty`` in the search."""

    def __init__(self, n_vocab: int):
        self.n = n_vocab

    def batch_score(self, ys, states, xs):
        return torch.ones(1, dtype=torch.float32, device=ys.device).expand(ys.shape[0], self.n), None


class _Running:
    """The hypotheses still being extended.  They advance in lock step, so all rows of ``yseq`` have the same length."""

    __slots__ = ("yseq", "score", "scores", "states")

    def __init__(self, yseq, score, scores, states):
        self.yseq, self.score, self.scores, self.states = yseq, score, scores, states

    def __len__(self):
        return self.yseq.shape[0]


def _end_detect(ended: List[Hypothesis], i: int, m_steps: int = 3, d_end: float = math.log(1 * math.exp(-10))) -> bool:
    """e2e_asr_common.py:14-44: stop when, for the last ``m_steps`` lengths, the best ended hypothesis of that length is far below the best."""
    if not ended:
        return False
    best = max(float(h.score) for h in ended)
    count = 0
    for m in range(m_steps):
        same = [float(h.score) for h in ended if len(h.yseq) == i - m]
        if same and max(same) - best < d_end:
            count += 1
    return count == m_steps


class BatchBeamSearchOnline:
    def __init__(self, scorers: Dict[str, Any], weights: Dict[str, float], beam_size: int, vocab_size: int, sos: int, eos: int,
                 token_list: Optional[List[str]] = None, pre_beam_ratio: float = 1.5, pre_beam_score_key: Optional[str] = None,
                 normalize_length: bool = False, block_size: int = 40, hop_size: int = 16, look_ahead: int = 16,
                 disable_repetition_detection: bool = False, encoded_feat_length_limit: int = 0, decoder_text_length_limit: int = 0,
                 incremental_decode: bool = False, time_sync: bool = False, **unused):
        if time_sync or block_size <= 0 or encoded_feat_length_limit or decoder_text_length_limit:
            raise NotImplementedError("espnet_b200.BatchBeamSearchOnline: block-wise search only (no time_sync, block_size 0 or length limits)")
        # scorers with weight 0 or None do not take part (beam_search.py:66-91); partial scorers are those with batch_score_partial
        self.weights, self.scorers, self.full, self.part = {}, {}, {}, {}
        for k, v in scorers.items():
            w = weights.get(k, 0)
            if w == 0 or v is None:
                continue
            self.weights[k], self.scorers[k] = w, v
            (self.part if hasattr(v, "batch_score_partial") else self.full)[k] = v
        self.sos, self.eos, self.n_vocab, self.token_list = sos, eos, vocab_size, token_list
        self.beam_size = beam_size
        self.pre_beam_size = int(pre_beam_ratio * beam_size)
        self.pre_beam_score_key = pre_beam_score_key
        if pre_beam_score_key is not None and pre_beam_score_key != "full" and pre_beam_score_key not in self.full:
            raise KeyError(f"{pre_beam_score_key} is not found in {list(self.full)}")
        self.do_pre_beam = pre_beam_score_key is not None and self.pre_beam_size < vocab_size and len(self.part) > 0
        self.normalize_length = normalize_length
        self.block_size, self.hop_size, self.look_ahead = block_size, hop_size, look_ahead
        self.disable_repetition_detection, self.incremental_decode = disable_repetition_detection, incremental_decode
        self.reset()

    def reset(self):
        self.encbuffer = None
        self.running: Optional[_Running] = None
        self.prev: Optional[_Running] = None
        self.ended: List[Hypothesis] = []
        self.processed_block = 0
        self.process_idx = 0
        self.prev_output = None

    # ------------------------------------------------------------------ hypothesis bookkeeping
    def _init(self, h: torch.Tensor) -> _Running:
        dev = h.device
        states = {k: [d.batch_init_state(h)] for k, d in self.scorers.items()}
        return _Running(torch.tensor([[self.sos]], dtype=torch.long, device=dev), torch.zeros(1, device=dev),
                        {k: torch.zeros(1, device=dev) for k in self.scorers}, states)

    def _pick(self, r: _Running, i: int) -> Hypothesis:
        return Hypothesis(yseq=r.yseq[i], score=r.score[i], scores={k: v[i] for k, v in r.scores.items()},
                          states={k: self.scorers[k].select_state(v, i) for k, v in r.states.items()})

    def _subset(self, r: _Running, ids: List[int]) -> _Running:
        idx = torch.tensor(ids, dtype=torch.long, device=r.yseq.device)
        return _Running(r.yseq[idx], r.score[idx], {k: v[idx] for k, v in r.scores.items()},
                        {k: [self.scorers[k].select_state(v, i) for i in ids] for k, v in r.states.items()})

    # ------------------------------------------------------------------ one search step (batch_beam_search.py:253-361)
    @torch.no_grad()
    def _step(self, r: _Running, h: torch.Tensor) -> _Running:
        n = len(r)
        xs = h.unsqueeze(0).expand(n, *h.shape)
        total = torch.zeros(n, self.n_vocab, dtype=torch.float32, device=h.device)
        sc, st = {}, {}
        for k, d in self.full.items():
            sc[k], st[k] = d.batch_score(r.yseq, r.states[k], xs)
            total += self.weights[k] * sc[k]
        part_ids = None
        if self.do_pre_beam:
            pre = total if self.pre_beam_score_key == "full" else sc[self.pre_beam_score_key]
            part_ids = torch.topk(pre, self.pre_beam_size, dim=-1)[1]
        for k, d in self.part.items():
            sc[k], st[k] = d.batch_score_partial(r.yseq, part_ids, r.states[k], h)
            total += self.weights[k] * sc[k]
        total += r.score.unsqueeze(1)
        top = total.view(-1).topk(self.beam_size)[1]
        parent, token = torch.div(top, self.n_vocab, rounding_mode="trunc"), top % self.n_vocab
        par, tok = parent.tolist(), token.tolist()
        states = {k: [d.select_state(st[k], p) for p in par] for k, d in self.full.items()}
        states.update({k: [d.select_state(st[k], p, t) for p, t in zip(par, tok)] for k, d in self.part.items()})
        return _Running(torch.cat([r.yseq[parent], token.unsqueeze(1)], dim=1), total[parent, token],
                        {k: r.scores[k][parent] + sc[k][parent, token] for k in self.scorers}, states)

    def _retire(self, i: int, maxlen: int, minlen: int, best: _Running) -> _Running:
        """batch_beam_search.py:363-423: at the last position every hypothesis is closed with <eos> (in place: the caller looks at ``best``
        again); hypotheses ending in <eos> move to the ended list (if long enough), the others keep running."""
        if i == maxlen - 1:
            logging.info("adding <eos> in the last position in the loop")
            best.yseq = torch.cat([best.yseq, torch.full((len(best), 1), self.eos, dtype=torch.long, device=best.yseq.device)], dim=1)
        is_eos = (best.yseq[:, -1] == self.eos).tolist()
        for b, e in enumerate(is_eos):
            if e and i >= minlen:
                self.ended.append(self._pick(best, b))
        return self._subset(best, [b for b, e in enumerate(is_eos) if not e])

    def _nbest(self, ended: List[Hypothesis]) -> List[Hypothesis]:
        key = (lambda h: float(h.score) / (len(h.yseq) - 1)) if self.normalize_length else (lambda h: float(h.score))
        out = sorted(ended, key=key, reverse=True)
        if not out:
            logging.warning("there is no N-best results, perform recognition again with smaller minlenratio.")
            return []
        best = out[0]
        for k, v in best.scores.items():
            logging.info(f"{float(v):6.2f} * {self.weights[k]:3} = {float(v) * self.weights[k]:6.2f} for {k}")
        logging.info(f"total log probability: {float(best.score):.2f}")
        logging.info(f"normalized log probability: {float(best.score) / len(best.yseq):.2f}")
        logging.info(f"total number of ended hypotheses: {len(out)}")
        if self.token_list is not None:
            logging.info("best hypo: " + "".join(self.token_list[int(t)] for t in best.yseq[1:-1]) + "\n")
        return out

    def extend(self, h: torch.Tensor, r: _Running):
        """Grow the scorers that keep per-frame quantities (the CTC prefix scorer) to the longer encoder output."""
        for k, d in self.scorers.items():
            if hasattr(d, "extend_prob"):
                d.extend_prob(h)
            if hasattr(d, "extend_state"):
                r.states[k] = d.extend_state(r.states[k])

    # ------------------------------------------------------------------ one block (batch_beam_search_online.py:389-487)
    def _process_block(self, h: torch.Tensor, is_final: bool, maxlen: int, minlen: int, maxlenratio: float) -> List[Hypothesis]:
        self.extend(h, self.running)
        local_ended: List[Hypothesis] = []
        while self.process_idx < maxlen:
            best = self._step(self.running, h)
            if self.process_idx == maxlen - 1:
                self.running = self._retire(self.process_idx, maxlen, minlen, best)
            last = best.yseq[:, -1]
            hit_eos = (last == self.eos).tolist()
            local_ended = [self._pick(best, i) for i, e in enumerate(hit_eos) if e]
            # a repeated token in a hypothesis that has not ended: the decoder is past the end of the block (Eq. 11 of the paper, implicit form)
            repeated = False
            if not self.disable_repetition_detection and not is_final:
                rep = (best.yseq[:, :-1] == last.unsqueeze(1)).any(dim=1).tolist()
                repeated = any(rp and not e for rp, e in zip(rep, hit_eos))
            if repeated:
                logging.info("Detected repetition.")
                break
            if is_final and maxlenratio == 0.0 and _end_detect(self.ended, self.process_idx):
                logging.info(f"end detected at {self.process_idx}")
                return self._nbest(self.ended)
            if local_ended and not is_final:
                logging.info("Detected hyp(s) reaching EOS in this block.")
                break
            self.prev = self.running
            self.running = self._retire(self.process_idx, maxlen, minlen, best)
            if is_final:
                self.ended.extend(local_ended)
            if len(self.running) == 0:
                logging.info("no hypothesis. Finish decoding.")
                return self._nbest(self.ended)
            self.process_idx += 1
        if is_final:
            return self._nbest(self.ended)
        rets = self._nbest(local_ended + self.ended)
        if self.process_idx > 1 and self.prev is not None and len(self.prev) > 0:   # rewind one step: the last expansion saw too little audio
            self.running, self.prev = self.prev, None
            self.process_idx -= 1
        return rets

    # ------------------------------------------------------------------ entry point (batch_beam_search_online.py:155-377, block-wise branch)
    @torch.no_grad()
    def __call__(self, x: torch.Tensor, maxlenratio: float = 0.0, minlenratio: float = 0.0, is_final: bool = True) -> List[Hypothesis]:
        """x (T, D): the encoder frames of this push.  Returns the n-best of the hypotheses ended so far ([] while nothing has ended yet)."""
        self.encbuffer = x if self.encbuffer is None else torch.cat([self.encbuffer, x], dim=0)
        x = self.encbuffer
        maxlen = x.shape[0] if maxlenratio == 0 else max(1, int(maxlenratio * x.shape[0]))
        minlen = -int(minlenratio) if minlenratio < 0 else int(minlenratio * x.shape[0])
        ret = None
        while True:
            end = self.block_size - self.look_ahead + self.hop_size * self.processed_block
            if end < x.shape[0]:
                h, block_is_final = x.narrow(0, 0, end), False
            elif is_final:
                h, block_is_final = x, True
            else:
                break
            if self.running is None:
                self.running = self._init(h)
            ret = self._process_block(h, block_is_final, maxlen, minlen, maxlenratio)
            self.processed_block += 1
            if self.incremental_decode and len(self.running) > 0:
                self.running = self._subset(self.running, [0])
            if block_is_final:
                return ret
        if ret is None:
            return [] if self.prev_output is None else self.prev_output
        self.prev_output = ret
        return ret

    forward = __call__
