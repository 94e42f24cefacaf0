"""Token-id / token / text conversion on the output side of Speech2Text (host-only; nothing here touches the GPU).

Reference: espnet2/text/token_id_converter.py:8-59 (TokenIDConverter), espnet2/text/build_tokenizer.py:17-100,
char_tokenizer.py:68-70, word_tokenizer.py:51-56, sentencepiece_tokenizer.py:35-37 (tokens2text), and the selection rule of
espnet2/bin/asr_inference.py:395-430 (token_type / bpemodel default to the training config; bpe without a model -> no tokenizer).
Only the decode direction used by inference is provided.
"""
from pathlib import Path
from typing import Iterable, List, Optional, Union

import numpy as np


def _read_token_file(path) -> List[str]:
    """One token per line; only the line terminator / trailing blanks are stripped, so a token that IS a leading space symbol survives."""
    return [ln[:1] + ln[1:].rstrip() for ln in Path(path).read_text(encoding="utf-8").splitlines(keepends=True)]


class TokenIDConverter:
    """id <-> token table with the reference's interface (token_list, token2id, unk_id, ids2tokens, tokens2ids, get_num_vocabulary_size) and
    its error conditions (duplicated symbol, missing unknown symbol: RuntimeError; non-1-D id array: ValueError)."""

    def __init__(self, token_list: Union[Path, str, Iterable[str]], unk_symbol: str = "<unk>"):
        self.token_list: List[str] = _read_token_file(token_list) if isinstance(token_list, (Path, str)) else list(token_list)
        self.token2id = {t: i for i, t in enumerate(self.token_list)}
        if len(self.token2id) != len(self.token_list):
            seen = set()
            dup = next(t for t in self.token_list if t in seen or seen.add(t))
            raise RuntimeError(f'Symbol "{dup}" is duplicated')
        if unk_symbol not in self.token2id:
            raise RuntimeError(f"Unknown symbol '{unk_symbol}' doesn't exist in the token_list")
        self.unk_symbol, self.unk_id = unk_symbol, self.token2id[unk_symbol]

    def get_num_vocabulary_size(self) -> int:
        return len(self.token_list)

    def ids2tokens(self, integers: Union[np.ndarray, Iterable[int]]) -> List[str]:
        if getattr(integers, "ndim", 1) != 1:
            raise ValueError(f"Must be 1 dim ndarray, but got {integers.ndim}")
        table = self.token_list
        return [table[int(i)] for i in integers]

    def tokens2ids(self, tokens: Iterable[str]) -> List[int]:
        lookup, unk = self.token2id.get, self.unk_id
        return [lookup(t, unk) for t in tokens]


class CharTokenizer:
    def __init__(self, space_symbol: str = "<space>"):
        self.space_symbol = space_symbol

    def __repr__(self):
        return f'{self.__class__.__name__}(space_symbol="{self.space_symbol}")'

    def text2tokens(self, line: str) -> List[str]:
        """char_tokenizer.py:48-66 without non-linguistic symbols: one token per character, " " -> space_symbol."""
        return [c if c != " " else self.space_symbol for c in line]

    def tokens2text(self, tokens: Iterable[str]) -> str:
        return "".join(t if t != self.space_symbol else " " for t in tokens)


class WordTokenizer:
    def __init__(self, delimiter: Optional[str] = None):
        self.delimiter = delimiter

    def __repr__(self):
        return f'{self.__class__.__name__}(delimiter="{self.delimiter}")'

    def text2tokens(self, line: str) -> List[str]:
        return line.split(self.delimiter)

    def tokens2text(self, tokens: Iterable[str]) -> str:
        return (" " if self.delimiter is None else self.delimiter).join(tokens)


class SentencepiecesTokenizer:
    """Lazy SentencePieceProcessor like the reference (the processor is not picklable)."""

    def __init__(self, model: Union[Path, str]):
        self.model = str(model)
        self.sp = None

    def __repr__(self):
        return f'{self.__class__.__name__}(model="{self.model}")'

    def _build(self):
        if self.sp is None:
            import sentencepiece as spm

            self.sp = spm.SentencePieceProcessor()
            self.sp.load(self.model)

    def text2tokens(self, line: str) -> List[str]:
        self._build()
        return self.sp.EncodeAsPieces(line)

    def tokens2text(self, tokens: Iterable[str]) -> str:
        self._build()
        return self.sp.DecodePieces(list(tokens))


def build_tokenizer(token_type: str, bpemodel: Union[Path, str, None] = None, space_symbol: str = "<space>",
                    delimiter: Optional[str] = None):
    if token_type == "bpe":
        if bpemodel is None:
            raise ValueError('bpemodel is required if token_type = "bpe"')
        return SentencepiecesTokenizer(bpemodel)
    if token_type == "word":
        return WordTokenizer(delimiter=delimiter)
    if token_type == "char":
        return CharTokenizer(space_symbol=space_symbol)
    raise NotImplementedError(f"espnet_b200: token_type {token_type!r} (supported: char, word, bpe)")


def tokenizer_for_inference(token_type: Optional[str], bpemodel, train_args):
    """asr_inference.py:395-430: explicit arguments win, else the training config; None / bpe-without-model -> no text output."""
    if token_type is None:
        token_type = getattr(train_args, "token_type", None)
    if bpemodel is None:
        bpemodel = getattr(train_args, "bpemodel", None)
    if token_type is None:
        return None
    if token_type == "bpe":
        return build_tokenizer("bpe", bpemodel) if bpemodel is not None else None
    return build_tokenizer(token_type, bpemodel)
