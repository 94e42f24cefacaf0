"""Speech2Text: the reference's inference entry class (espnet2/bin/asr_inference.py:73-677) over the
espnet_b200 CUDA path, plus the model container / registries it needs (espnet2/asr/espnet_model.py:380-467,
espnet2/tasks/asr.py:95-206,512-651).

Same constructor keywords that matter for this path (asr_train_config, asr_model_file, device, dtype,
beam_size, ctc_weight, penalty, nbest, maxlenratio, minlenratio, normalize_length), same
``__call__(speech) -> [(text, token, token_int, Hypothesis)]``, same attributes (``asr_model``,
``asr_train_args``, ``beam_search``, ``converter``, ``tokenizer``).  Extension: ``batch_decode(list)``
decodes many utterances in one pass (the reference is batch-1; ESPnet3's runner passes lists,
espnet3/systems/base/inference_runner.py:262-275).
"""
import argparse
import logging
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import yaml

from . import lib
from .branchformer_encoder import BranchformerEncoder
from .ctc import CTC
from .decoder import TransformerDecoder
from .e_branchformer_encoder import EBranchformerEncoder
from .encoder import ConformerEncoder
from .errors import TooShortUttError  # noqa: F401
from .frontend import DefaultFrontend, GlobalMVN, UtteranceMVN
from .text import TokenIDConverter, tokenizer_for_inference
from .search import BatchBeamSearch, Hypothesis
from .transformer_encoder import TransformerEncoder

logger = logging.getLogger(__name__)

# name -> class registries, as espnet2/tasks/asr.py:95-206 (only the classes on the north-star path)
frontend_choices = {"default": DefaultFrontend}
normalize_choices = {"global_mvn": GlobalMVN, "utterance_mvn": UtteranceMVN}
from .streaming_encoder import ContextualBlockConformerEncoder, ContextualBlockTransformerEncoder  # noqa: E402

encoder_choices = {"conformer": ConformerEncoder, "transformer": TransformerEncoder, "contextual_block_conformer": ContextualBlockConformerEncoder,
                   "contextual_block_transformer": ContextualBlockTransformerEncoder, "e_branchformer": EBranchformerEncoder, "branchformer": BranchformerEncoder}
decoder_choices = {"transformer": TransformerDecoder}


class ESPnetASRModel(torch.nn.Module):
    """frontend -> normalize -> encoder (+ decoder, ctc): the encode() half of espnet_model.py:380-467."""

    def __init__(self, vocab_size, token_list, frontend, normalize, encoder, decoder, ctc, ctc_weight=0.5, sym_blank="<blank>"):
        super().__init__()
        self.blank_id = list(token_list).index(sym_blank) if sym_blank in token_list else 0
        self.sos = self.eos = vocab_size - 1  # espnet_model.py:76-87
        self.vocab_size, self.token_list = vocab_size, list(token_list)
        self.frontend, self.normalize, self.encoder = frontend, normalize, encoder
        self.decoder = decoder
        self.ctc = ctc
        self.ctc_weight = ctc_weight

    @torch.no_grad()
    def encode(self, speech: torch.Tensor, speech_lengths: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """speech (B, L) CUDA float32, speech_lengths (B,) -> (B, T, D), (B,)."""
        speech = speech[:, : int(speech_lengths.max())]
        feats, feats_lengths = self.frontend(speech, speech_lengths)
        if self.normalize is not None:
            feats, feats_lengths = self.normalize(feats, feats_lengths)
        enc, enc_lens, _ = self.encoder(feats, feats_lengths)
        return enc, enc_lens

    def enc_split(self, enc):
        """tf32 hi/lo copy of the encoder output made by its last LayerNorm (avoids a re-split pass)."""
        ls = self.encoder.last_split_out
        return ls[1] if ls is not None and ls[0] == enc.data_ptr() else None


def build_model(args: argparse.Namespace) -> ESPnetASRModel:
    """ASRTask.build_model (espnet2/tasks/asr.py:512-651) for the supported classes."""
    token_list = list(args.token_list)
    vocab_size = len(token_list)
    # SpecAug (specaug: specaug) augments only in training (espnet_model.py:394) and has no parameters or buffers: every recipe-written
    # config.yaml names it, so it is accepted and specaug_conf ignored
    if getattr(args, "specaug", None) not in (None, "specaug"):
        raise NotImplementedError(f"specaug={args.specaug} is not on the espnet_b200 inference path")
    for key in ("preencoder", "postencoder"):
        if getattr(args, key, None) is not None:
            raise NotImplementedError(f"{key} is not on the espnet_b200 inference path")
    if getattr(args, "input_size", None) is not None:
        raise NotImplementedError("input_size != None (pre-extracted features): use the frontend")
    frontend = frontend_choices[args.frontend](**(args.frontend_conf or {}))
    input_size = frontend.output_size()
    normalize = None
    if getattr(args, "normalize", None) is not None:
        normalize = normalize_choices[args.normalize](**(args.normalize_conf or {}))
    encoder = encoder_choices[args.encoder](input_size=input_size, **(args.encoder_conf or {}))
    decoder = None
    if getattr(args, "decoder", None) is not None:
        decoder = decoder_choices[args.decoder](vocab_size=vocab_size, encoder_output_size=encoder.output_size(),
                                                **(args.decoder_conf or {}))
    ctc = CTC(odim=vocab_size, encoder_output_size=encoder.output_size(), **(getattr(args, "ctc_conf", None) or {}))
    mc = dict(getattr(args, "model_conf", None) or {})
    return ESPnetASRModel(vocab_size, token_list, frontend, normalize, encoder, decoder, ctc, ctc_weight=mc.get("ctc_weight", 0.5))


def build_model_from_file(config_file, model_file=None, device="cuda"):
    """AbsTask.build_model_from_file (espnet2/tasks/abs_task.py:2456-2561): yaml -> Namespace -> model -> load_state_dict."""
    with open(config_file, "r", encoding="utf-8") as f:
        args = argparse.Namespace(**yaml.safe_load(f))
    model = build_model(args).to(device)
    if model_file is not None:
        sd = torch.load(model_file, map_location=device)
        for k in ("module", "state_dict"):
            if isinstance(sd, dict) and k in sd and isinstance(sd[k], dict):
                sd = sd[k]
        model.load_state_dict(sd, strict=False)
    return model, args


# keywords of the reference constructor that would change the result if honoured (refused unless left at their defaults) ...
_REFUSED_KWARGS = {"ngram_file", "transducer_conf", "streaming", "quantize_asr_model", "quantize_lm",
                   "enh_s2t_task", "hugging_face_decoder", "multi_asr", "partial_ar", "lid_prompt",
                   "lang_prompt_token", "nlp_prompt_token", "prompt_token_file", "time_sync"}
# ... and those that cannot (accepted without a warning)
_HARMLESS_KWARGS = {"ngram_scorer", "quantize_modules", "quantize_dtype", "search_beam_size", "decoder_text_length_limit", "encoded_feat_length_limit", "hugging_face_decoder_conf",
                    "threshold_probability", "max_seq_len", "max_mask_parallel"}


class Speech2Text:
    def __init__(self, asr_train_config=None, asr_model_file=None, device: str = "cuda", dtype: str = "float32",
                 beam_size: int = 20, ctc_weight: float = 0.5, lm_weight: float = 1.0, ngram_weight: float = 0.9,
                 penalty: float = 0.0, nbest: int = 1, maxlenratio: float = 0.0, minlenratio: float = 0.0,
                 normalize_length: bool = False, batch_size: int = 1, token_type: Optional[str] = None, bpemodel: Optional[str] = None,
                 asr_model: Optional[ESPnetASRModel] = None, asr_train_args=None, lm_train_config=None, lm_file=None, lm=None, **unused):
        if dtype != "float32":
            raise NotImplementedError("espnet_b200 computes in float32 (the reference's inference dtype)")
        # Reference keywords (asr_inference.py:86-127) that select a different decoding algorithm must not be dropped silently.
        refused = {k: v for k, v in unused.items()
                   if k in _REFUSED_KWARGS and v not in (None, False, "", {}, [])}
        if refused:
            raise NotImplementedError("espnet_b200.Speech2Text does not implement: " + ", ".join(f"{k}={v!r}" for k, v in sorted(refused.items())))
        ignored = sorted(k for k in unused if k not in _REFUSED_KWARGS and k not in _HARMLESS_KWARGS)
        if ignored:
            logger.warning("espnet_b200.Speech2Text ignores these keyword arguments: " + ", ".join(ignored))
        if not str(device).startswith("cuda"):
            raise RuntimeError("espnet_b200 has no CPU path: device must be a CUDA device")
        lib.load()  # fail loudly if the CUDA library is missing
        if asr_model is None:
            asr_model, asr_train_args = build_model_from_file(asr_train_config, asr_model_file, device)
        if isinstance(asr_model.encoder, ContextualBlockTransformerEncoder):
            raise NotImplementedError("espnet_b200.Speech2Text: the contextual-block Transformer encoder is a streaming encoder (forward_infer "
                                      "returns no lengths); decode it with Speech2TextStreaming")
        asr_model = asr_model.to(device).eval()
        self.asr_model, self.asr_train_args = asr_model, asr_train_args
        self.device, self.dtype, self.nbest = device, dtype, nbest
        self.maxlenratio, self.minlenratio = maxlenratio, minlenratio
        token_list = asr_model.token_list
        decoder = asr_model.decoder if ctc_weight != 1.0 else None  # espnet_model.py:167-173
        scorers = dict(decoder=decoder, ctc=asr_model.ctc)
        if lm is None and lm_train_config is not None:      # LM shallow fusion (asr_inference.py:178-191): scorers["lm"] = lm.lm
            from .lm import build_lm_from_file

            lm, self.lm_train_args = build_lm_from_file(lm_train_config, lm_file, device)
        if lm is not None:
            scorers["lm"] = lm.to(device).eval()
        weights = dict(decoder=1.0 - ctc_weight, ctc=ctc_weight, lm=lm_weight, ngram=ngram_weight, length_bonus=penalty)
        self.beam_search = BatchBeamSearch(scorers, weights, beam_size, len(token_list), asr_model.sos, asr_model.eos,
                                           token_list=token_list, pre_beam_score_key=None if ctc_weight == 1.0 else "full",
                                           normalize_length=normalize_length)
        self.converter = TokenIDConverter(token_list)
        self.tokenizer = tokenizer_for_inference(token_type, bpemodel, asr_train_args)   # asr_inference.py:395-430
        logger.info(f"Text tokenizer: {self.tokenizer}")

    @staticmethod
    def from_pretrained(model_tag: Optional[str] = None, **kwargs):
        """asr_inference.py:680-707: with a model tag the files come from espnet_model_zoo (must be installed, as for the reference)."""
        if model_tag is not None:
            try:
                from espnet_model_zoo.downloader import ModelDownloader
            except ImportError:
                logger.error("`espnet_model_zoo` is not installed. Please install via `pip install -U espnet_model_zoo`.")
                raise
            kwargs.update(**ModelDownloader().download_and_unpack(model_tag))
        return Speech2Text(**kwargs)

    def _to_batch(self, speeches: Sequence[Union[torch.Tensor, np.ndarray]]):
        lens = torch.tensor([int(s.shape[0]) for s in speeches], dtype=torch.long)
        L = int(lens.max())
        host = torch.zeros(len(speeches), L, dtype=torch.float32).pin_memory()
        for i, s in enumerate(speeches):
            host[i, : lens[i]] = torch.as_tensor(s, dtype=torch.float32)
        return host.to(self.device, non_blocking=True), lens

    def _log_best(self, nbest_hyps: List[Hypothesis]):
        """End-of-search log lines of beam_search.py:460-487 (utils/calculate_rtf.py pairs 'speech length' with 'best hypo')."""
        if not nbest_hyps:
            logger.warning("there is no N-best results")
            return
        best = nbest_hyps[0]
        w = self.beam_search.weights
        for k, v in best.scores.items():
            logger.info(f"{v:6.2f} * {w.get(k, 0.0):3} = {v * w.get(k, 0.0):6.2f} for {k}")
        logger.info(f"total log probability: {float(best.score):.2f}")
        logger.info(f"normalized log probability: {float(best.score) / len(best.yseq):.2f}")
        logger.info(f"total number of ended hypotheses: {len(nbest_hyps)}")
        logger.info("best hypo: " + "".join(self.converter.token_list[x] for x in best.yseq[1:-1].tolist()) + "\n")

    def _results(self, nbest_hyps: List[Hypothesis]):
        if logger.isEnabledFor(logging.INFO):
            self._log_best(nbest_hyps)
        results = []
        for hyp in nbest_hyps[: self.nbest]:
            token_int = hyp.yseq[1:-1].tolist()                       # asr_inference.py:659-666
            token_int = list(filter(lambda x: x != 0, token_int))
            token = self.converter.ids2tokens(token_int)
            text = self.tokenizer.tokens2text(token) if self.tokenizer is not None else None
            results.append((text, token, token_int, hyp))
        return results

    @torch.no_grad()
    def batch_decode(self, speeches: Sequence[Union[torch.Tensor, np.ndarray]]):
        """List of 1-D waveforms -> list of result lists (each as __call__ returns for one utterance)."""
        speech, lens = self._to_batch(speeches)
        enc, enc_lens = self.asr_model.encode(speech, lens)
        hyps = self.beam_search.forward_batch(enc, enc_lens, self.asr_model.enc_split(enc), self.maxlenratio, self.minlenratio)
        return [self._results(h) for h in hyps]

    @torch.no_grad()
    def batch_decode_padded(self, speech: torch.Tensor, lengths: torch.Tensor):
        """Pre-batched input: speech (B, Lmax) float32 (pinned host or device memory), lengths (B,) -> as batch_decode."""
        speech = speech.to(self.device, non_blocking=True)
        enc, enc_lens = self.asr_model.encode(speech, lengths)
        hyps = self.beam_search.forward_batch(enc, enc_lens, self.asr_model.enc_split(enc), self.maxlenratio, self.minlenratio)
        return [self._results(h) for h in hyps]

    @torch.no_grad()
    def batch_decode_sharded(self, speech: torch.Tensor, lengths: torch.Tensor, max_tokens: int = 256):
        """Utterance-sharded decoding over the ranks of an initialised torch.distributed job (one process per GPU; the reference shards by
        splitting the key file over processes, asr.sh:1591-1618): this rank decodes ITS utterances (speech (B_local, Lmax), pinned host or device)
        and every rank receives the n-best token ids and scores of all utterances -- one all-gather of fixed-width records, no other
        collective.  Returns (local results as batch_decode_padded, [rank][utterance][(token ids, score)])."""
        import torch.distributed as dist

        from . import sharding

        import os
        import time

        t0 = time.perf_counter()
        local = self.batch_decode_padded(speech, lengths)
        t1 = time.perf_counter()
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        out = local, sharding.all_gather_results(local, self.nbest, max_tokens, world, device=self.device)
        if os.environ.get("ESPB_BENCH_DEBUG"):
            logger.warning(f"batch_decode_sharded: decode {1e3 * (t1 - t0):.1f} ms, exchange {1e3 * (time.perf_counter() - t1):.1f} ms")
        return out

    def decode_stream(self, batches, sharded: bool = False):
        """Iterate over (speech (B, Lmax) pinned host memory, lengths) batches with the host-to-device copy of batch k+1 running on a copy
        stream under the computation of batch k (double buffering; the device buffer of a batch is released to the copy stream once its
        encoder pass has consumed it).  Yields what batch_decode_padded / batch_decode_sharded returns."""
        if getattr(self, "_copy_stream", None) is None:    # one copy stream per instance: the caching allocator pools blocks per stream
            self._copy_stream = torch.cuda.Stream(device=self.device)
        copy_stream = self._copy_stream
        main = torch.cuda.current_stream(self.device)

        def start(item):
            sp, ln = item
            with torch.cuda.stream(copy_stream):
                dev = sp.to(self.device, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(copy_stream)
            return dev, ln, ev

        it = iter(batches)
        try:
            nxt = start(next(it))
        except StopIteration:
            return
        while nxt is not None:
            dev, ln, ev = nxt
            main.wait_event(ev)
            dev.record_stream(main)
            try:
                nxt = start(next(it))
            except StopIteration:
                nxt = None
            yield self.batch_decode_sharded(dev, ln) if sharded else self.batch_decode_padded(dev, ln)

    @torch.no_grad()
    def __call__(self, speech: Union[torch.Tensor, np.ndarray]):
        logger.info("speech length: " + str(int(speech.shape[0])))
        return self.batch_decode([speech])[0]

    @torch.no_grad()
    def ctc_greedy(self, speeches: Sequence[Union[torch.Tensor, np.ndarray]]):
        """CTC.argmax -> unique_consecutive -> drop blank (asr/ctc.py:207-215, s2t_inference_ctc.py:630-632), batched.
        Returns a list of python lists of token ids."""
        speech, lens = self._to_batch(speeches)
        enc, enc_lens = self.asr_model.encode(speech, lens)
        ids, cnt, _ = self.asr_model.ctc.greedy(enc, enc_lens, self.asr_model.enc_split(enc), blank=self.asr_model.blank_id)
        ids, cnt = ids.cpu(), cnt.cpu()
        return [ids[b, : int(cnt[b])].tolist() for b in range(ids.shape[0])]
