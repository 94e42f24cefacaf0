"""Perplexity of a language model over text sets: espnet2/bin/lm_calc_perplexity.py ``calc_perplexity`` on the CUDA path.

Reads ``key text`` files (the ``text`` type of the reference's data loader), tokenises them with the LM's ``token_type`` / ``token_list``
(char, word or bpe, as the reference's CommonPreprocessor without cleaner, g2p or non-linguistic symbols), pads each batch with 0 (the LM
collate, tasks/lm.py:141-145), runs ``ESPnetLanguageModel.nll`` and writes what the reference writes: ``utt2ppl`` and ``utt2ntokens`` per
utterance, the corpus ``ppl`` and the logarithm ``base``.
"""
import logging
from pathlib import Path
from typing import Iterator, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .bin_asr_inference import ResultDirWriter
from .lm import build_espnet_lm_from_file
from .text import TokenIDConverter, build_tokenizer


def read_text(path: str, key_file: Optional[str] = None) -> Iterator[Tuple[str, str]]:
    """(key, text) of a ``key text`` file, restricted to the keys of key_file if given; a line without text is refused, as the reference's
    streaming loader refuses it (iterable_dataset.py:190-195)."""
    keep = None
    if key_file is not None:
        with open(key_file, encoding="utf-8") as f:
            keep = {ln.split(maxsplit=1)[0] for ln in f if ln.strip()}
    with open(path, encoding="utf-8") as f:
        for ln in f:
            sps = ln.rstrip().split(maxsplit=1)
            if len(sps) != 2:
                raise RuntimeError(f"This line doesn't include a space: {path}: {ln!r}")
            key, text = sps
            if keep is None or key in keep:
                yield key, text


def text_to_ids(train_args):
    """CommonPreprocessor's text branch (espnet2/train/preprocessor.py) for the LM's config -> a function text -> token ids."""
    if not getattr(train_args, "use_preprocessor", True):
        raise NotImplementedError("espnet_b200 lm_calc_perplexity tokenises the text: the LM config needs use_preprocessor: true")
    for opt in ("cleaner", "g2p", "non_linguistic_symbols"):
        if getattr(train_args, opt, None) is not None:
            raise NotImplementedError(f"espnet_b200 lm_calc_perplexity: {opt} is not supported (got {getattr(train_args, opt)!r})")
    tokenizer = build_tokenizer(getattr(train_args, "token_type", None), getattr(train_args, "bpemodel", None))
    converter = TokenIDConverter(train_args.token_list)
    return lambda text: converter.tokens2ids(tokenizer.text2tokens(text))


def _perplexity(nll, ntokens, log_base):
    if log_base is None:
        return np.exp(nll / ntokens)
    return log_base ** (nll / ntokens / np.log(log_base))


def calc_perplexity(output_dir: str, batch_size: int, dtype: str, ngpu: int, seed: int, num_workers: int, log_level: Union[int, str],
                    data_path_and_name_and_type: Sequence[Tuple[str, str, str]], key_file: Optional[str], train_config: Optional[str],
                    model_file: Optional[str], log_base: Optional[float], allow_variable_data_keys: bool):
    """lm_calc_perplexity.py:23-131 with the same arguments.  ngpu 0 is refused (there is no CPU path); ngpu > 1 runs on one GPU."""
    logging.basicConfig(level=log_level, format="%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s")
    if dtype != "float32":
        raise NotImplementedError(f"espnet_b200 computes in float32 (dtype {dtype!r} requested)")
    if ngpu < 1:
        raise RuntimeError("espnet_b200 runs on the GPU only: ngpu must be >= 1")
    texts = [d for d in data_path_and_name_and_type if d[1] == "text"]
    if len(texts) != 1 or any(d[2] != "text" for d in texts) or (len(data_path_and_name_and_type) > 1 and not allow_variable_data_keys):
        raise NotImplementedError("espnet_b200 lm_calc_perplexity reads one (path, 'text', 'text') input")
    torch.manual_seed(seed)
    np.random.seed(seed)

    model, train_args = build_espnet_lm_from_file(train_config, model_file, "cuda")
    to_ids = text_to_ids(train_args)
    items = [(k, to_ids(t)) for k, t in read_text(texts[0][0], key_file)]

    with ResultDirWriter(output_dir) as writer:
        total_nll, total_ntokens = 0.0, 0
        for i in range(0, len(items), batch_size):
            keys = [k for k, _ in items[i:i + batch_size]]
            seqs: List[List[int]] = [ids for _, ids in items[i:i + batch_size]]
            lengths = torch.tensor([len(s) for s in seqs], dtype=torch.long)
            text = torch.zeros(len(seqs), max(1, int(lengths.max())), dtype=torch.long)   # CommonCollateFn(int_pad_value=0)
            for b, s in enumerate(seqs):
                text[b, :len(s)] = torch.tensor(s, dtype=torch.long)
            nll, x_lengths = model.nll(text, lengths)
            nll = nll.detach().cpu().numpy().sum(1)           # float32 sums, as the reference's
            x_lengths = x_lengths.detach().cpu().numpy()
            total_nll += nll.sum()
            total_ntokens += x_lengths.sum()
            for key, _nll, ntoken in zip(keys, nll, x_lengths):
                writer["utt2ppl"][key] = str(_perplexity(_nll, ntoken, log_base))
                writer["utt2ntokens"][key] = str(ntoken)

        ppl = _perplexity(total_nll, total_ntokens, log_base)
        with (Path(output_dir) / "ppl").open("w", encoding="utf-8") as f:
            f.write(f"{ppl}\n")
        with (Path(output_dir) / "base").open("w", encoding="utf-8") as f:
            f.write(f"{np.e if log_base is None else log_base}\n")
        logging.info(f"PPL={ppl}")
