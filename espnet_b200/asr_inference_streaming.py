"""Speech2TextStreaming for N live streams in lock step: chunked frontend -> contextual-block encoder -> block-synchronous beam search
(SURVEY.md 8f-2, BASELINE configs[3]).

Reference: espnet2/bin/asr_inference_streaming.py:35-357.  ``apply_frontend`` is the reference's algorithm (waveform overlap buffer of
(2*ceil(ceil(win/hop)/2) - 1) hops + residual, STFT of the buffered chunk, trimming of the ceil(ceil(win/hop)/2) edge frames) with a leading
stream dimension: every stream pushes the same number of samples per call, so one (N, n) tensor replaces N Python objects.  The encoder is
``ContextualBlockConformerEncoder.forward_infer`` or ``ContextualBlockTransformerEncoder.forward_infer`` (streaming_encoder.py), batched over
the streams; only its outputs are read, not its lengths (the Transformer returns None there, as the reference).

Decoding: as the reference, every push hands the new encoder frames of a stream to its ``BatchBeamSearchOnline`` (search_online.py: joint CTC /
attention (/ LM) block-synchronous beam search, one search object per stream, the decoder and LM shared) and returns
``[(text, token, token_int, Hypothesis)]`` of the hypotheses ended so far.  ``greedy=True`` replaces the search by incremental CTC-greedy output
(argmax -> collapse repeats across pushes -> drop blank, as asr/ctc.py:207-215 does for whole utterances): the throughput mode of ``bench.py``.
"""
import math
from typing import List, Optional

import torch

from . import ops
from .lib import call, ptr
from .ops import _count


class Speech2TextStreaming:
    def __init__(self, asr_model=None, n_streams: int = 1, device: str = "cuda", ctc_weight: float = 0.5, asr_train_config=None,
                 asr_model_file=None, lm_train_config=None, lm_file=None, lm=None, token_type: Optional[str] = None, bpemodel: Optional[str] = None,
                 beam_size: int = 20, lm_weight: float = 1.0, penalty: float = 0.0, nbest: int = 1, maxlenratio: float = 0.0,
                 minlenratio: float = 0.0, normalize_length: bool = False, disable_repetition_detection: bool = False,
                 decoder_text_length_limit: int = 0, encoded_feat_length_limit: int = 0, batch_size: int = 1, dtype: str = "float32",
                 greedy: bool = False, **unused):
        """``asr_model``: a built ESPnetASRModel, or -- as the reference's constructor (asr_inference_streaming.py:46-75) -- ``asr_train_config`` (+
        ``asr_model_file``) to build it from the reference's own config.yaml / checkpoint."""
        if dtype != "float32":
            raise NotImplementedError("espnet_b200 computes in float32 (the reference's inference dtype)")
        if batch_size != 1:
            raise NotImplementedError("batch decoding is not implemented (as the reference): push N streams as an (N, n) tensor instead")
        asr_train_args = None
        if asr_model is None or isinstance(asr_model, (str, bytes)) or hasattr(asr_model, "__fspath__"):
            from .asr_inference import build_model_from_file

            cfg = asr_train_config if asr_model is None else asr_model
            if cfg is None:
                raise ValueError("Speech2TextStreaming needs asr_model or asr_train_config")
            asr_model, asr_train_args = build_model_from_file(cfg, asr_model_file, device)
        self.asr_model = asr_model.to(device).eval()
        self.device, self.n = device, n_streams
        fe = asr_model.frontend
        self.hop_length, self.win_length = fe.hop_length, fe.win_length
        self.edge = math.ceil(math.ceil(self.win_length / self.hop_length) / 2)      # frames trimmed at a chunk edge
        self.blank = asr_model.blank_id
        self.greedy, self.nbest, self.maxlenratio, self.minlenratio = greedy, nbest, maxlenratio, minlenratio
        self.searches = None
        if not greedy:
            from .ctc import CTCPrefixScorer
            from .search_online import BatchBeamSearchOnline, LengthBonus
            from .text import TokenIDConverter, tokenizer_for_inference

            if lm is None and lm_train_config is not None:
                from .lm import build_lm_from_file

                lm, _ = build_lm_from_file(lm_train_config, lm_file, device)
            token_list = asr_model.token_list
            ecfg = getattr(asr_train_args, "encoder_conf", None) or {}
            enc = asr_model.encoder
            blk = {k: ecfg.get(k, getattr(enc, k)) for k in ("block_size", "hop_size", "look_ahead")}
            weights = dict(decoder=1.0 - ctc_weight, ctc=ctc_weight, lm=lm_weight, length_bonus=penalty)   # asr_inference_streaming.py:105-110
            self.searches = []
            for _ in range(n_streams):       # the CTC prefix scorer keeps the posteriors of its stream; decoder and LM are stateless across calls
                scorers = dict(decoder=asr_model.decoder, ctc=CTCPrefixScorer(asr_model.ctc, asr_model.eos), length_bonus=LengthBonus(len(token_list)))
                if lm is not None:
                    scorers["lm"] = lm.to(device).eval()
                self.searches.append(BatchBeamSearchOnline(
                    scorers, weights, beam_size, len(token_list), asr_model.sos, asr_model.eos, token_list=token_list,
                    pre_beam_score_key=None if ctc_weight == 1.0 else "full", normalize_length=normalize_length,
                    disable_repetition_detection=disable_repetition_detection, decoder_text_length_limit=decoder_text_length_limit,
                    encoded_feat_length_limit=encoded_feat_length_limit, **blk))
            self.converter = TokenIDConverter(token_list)
            self.tokenizer = tokenizer_for_inference(token_type, bpemodel, asr_train_args)
        self.reset()

    def reset(self):
        self.frontend_states, self.encoder_states = None, None
        self.last_tok = torch.full((self.n,), -1, dtype=torch.int32, device=self.device)    # previous frame's argmax per stream (collapse across pushes)
        self.tokens: List[List[int]] = [[] for _ in range(self.n)]
        for bs in self.searches or []:
            bs.reset()

    @torch.no_grad()
    def apply_frontend(self, speech: torch.Tensor, prev_states=None, is_final: bool = False):
        """speech (N, n) float32 -> (feats (N, T, n_mels) | None, next_states)   [asr_inference_streaming.py:205-294]"""
        speech = speech.to(self.device, non_blocking=True).float()
        if prev_states is not None:
            speech = torch.cat([prev_states["waveform_buffer"], speech], dim=1)
        n = speech.shape[1]
        if n <= self.win_length:
            if not is_final:
                return None, {"waveform_buffer": speech.clone()}
            speech = torch.cat([speech, speech.new_zeros(speech.shape[0], self.win_length - n)], dim=1)
            n = speech.shape[1]
        if is_final:
            to_process, buf = speech, None
        else:
            n_frames, n_res = n // self.hop_length, n % self.hop_length
            keep = (2 * self.edge - 1) * self.hop_length + n_res
            to_process = speech[:, : n_frames * self.hop_length]
            buf = speech[:, n - keep:].clone()
        to_process = to_process.contiguous()
        lens = torch.full((to_process.shape[0],), to_process.shape[1], dtype=torch.long)
        feats, flens = self.asr_model.frontend(to_process, lens)
        feats._espb_partial = None          # chunk statistics are not utterance statistics
        if self.asr_model.normalize is not None:
            feats, flens = self.asr_model.normalize(feats, flens)
        T = feats.shape[1]
        if is_final:
            if prev_states is not None:
                feats = feats[:, self.edge:]
        elif prev_states is None:
            feats = feats[:, : T - self.edge]
        else:
            feats = feats[:, self.edge: T - self.edge]
        return feats.contiguous(), (None if is_final else {"waveform_buffer": buf})

    def assemble_hyps(self, hyps):
        """asr_inference_streaming.py:337-357: n-best -> (text, token, token_int, hyp); <sos>/<eos> and blank (id 0) removed."""
        results = []
        for hyp in hyps[: self.nbest]:
            token_int = [t for t in hyp.yseq[1:-1].tolist() if t != 0]
            token = self.converter.ids2tokens(token_int)
            text = self.tokenizer.tokens2text(token) if self.tokenizer is not None else None
            results.append((text, token, token_int, hyp))
        return results

    @torch.no_grad()
    def __call__(self, speech, is_final: bool = False):
        """speech (N, n) -- or (n,) for one stream, as the reference -- : the next n samples of every stream.

        Beam-search mode: the reference's ``[(text, token, token_int, Hypothesis)]`` for a 1-D push, a list of those (one per stream) for an (N, n)
        push.  ``greedy=True``: per stream, the token ids this push added."""
        if not isinstance(speech, torch.Tensor):
            speech = torch.as_tensor(speech)
        single = speech.dim() == 1
        if single:
            speech = speech.unsqueeze(0)
        assert speech.dim() == 2 and speech.shape[0] == self.n
        feats, self.frontend_states = self.apply_frontend(speech, self.frontend_states, is_final)
        enc = None
        if feats is not None and feats.shape[1] > 0:
            lens = torch.full((self.n,), feats.shape[1], dtype=torch.long)
            enc, _, self.encoder_states = self.asr_model.encoder(feats, lens, self.encoder_states, is_final=is_final, infer_mode=True)
        if not self.greedy:
            ret = [[] for _ in range(self.n)]
            if feats is not None:           # (the reference searches whenever the frontend produced features, also over zero new frames)
                for s, bs in enumerate(self.searches):
                    x = enc[s] if enc is not None else torch.zeros(0, self.asr_model.encoder.output_size(), device=self.device)
                    ret[s] = self.assemble_hyps(bs(x=x, maxlenratio=self.maxlenratio, minlenratio=self.minlenratio, is_final=is_final))
            if is_final:
                self.reset()
            return ret[0] if single else ret
        new = [[] for _ in range(self.n)]
        if enc is not None and enc.shape[1] > 0:
            ctc = self.asr_model.ctc
            am = ctc.argmax(enc).to(torch.int32)                        # (N, T)
            prev = torch.cat([self.last_tok.view(-1, 1), am[:, :-1]], dim=1)
            keep = (am != prev) & (am != self.blank)
            self.last_tok = am[:, -1].contiguous()
            am_c, keep_c = am.cpu(), keep.cpu()
            for s in range(self.n):
                new[s] = am_c[s][keep_c[s]].tolist()
                self.tokens[s].extend(new[s])
        if is_final:
            done = [list(t) for t in self.tokens]
            self.reset()
            self.final_tokens = done
        return new
