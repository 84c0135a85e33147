"""BERT-uncased tokenization for InternVideo2's text tower, host side (no `transformers` import), in the spirit of models/clip.py.

What the reference's tokenizer does to a caption (get_txt_feat, cosmos_curate/models/internvideo2_mm.py:219-241: BertTokenizer of
google-bert/bert-large-uncased called with padding="max_length", truncation=True, max_length=40):
  * basic tokenization: drop NUL, U+FFFD and control characters and map whitespace to a space; put every CJK ideograph in a token
    of its own; split on whitespace; lower-case, NFD and drop combining marks (accents); split punctuation off;
  * WordPiece: greedy longest match first against vocab.txt, continuations prefixed "##"; a word longer than 100 characters, or
    one with no complete match, becomes [UNK];
  * [CLS] + pieces[:max_len - 2] + [SEP], then [PAD] up to max_len.
The special tokens ([CLS], [SEP], [PAD], [UNK], [MASK]) written literally in a text stay whole, as the reference keeps them.
"""

from __future__ import annotations

import re
import unicodedata
from pathlib import Path

import numpy as np

BERT_VOCAB_ID = "google-bert/bert-large-uncased"
SPECIAL_TOKENS = ("[UNK]", "[SEP]", "[PAD]", "[CLS]", "[MASK]")
MAX_WORD_CHARS = 100
_SPECIAL_RE = re.compile("(" + "|".join(re.escape(t) for t in SPECIAL_TOKENS) + ")")
# CJK ideograph blocks: Unified Ideographs, Extension A-E, Compatibility Ideographs and their supplement
_CJK = ((0x4E00, 0x9FFF), (0x3400, 0x4DBF), (0x20000, 0x2A6DF), (0x2A700, 0x2B73F), (0x2B740, 0x2B81F), (0x2B820, 0x2CEAF),
        (0xF900, 0xFAFF), (0x2F800, 0x2FA1F))  # fmt: skip


def _is_whitespace(ch: str) -> bool:
    return ch in " \t\n\r" or unicodedata.category(ch) == "Zs"


def _is_control(ch: str) -> bool:
    return ch not in "\t\n\r" and unicodedata.category(ch).startswith("C")


def _is_punctuation(ch: str) -> bool:
    cp = ord(ch)  # every non-alphanumeric printable ASCII character counts, e.g. "^", "$" and "`" (not Unicode P*)
    return 33 <= cp <= 47 or 58 <= cp <= 64 or 91 <= cp <= 96 or 123 <= cp <= 126 or unicodedata.category(ch).startswith("P")


def _is_cjk(ch: str) -> bool:
    cp = ord(ch)
    return any(lo <= cp <= hi for lo, hi in _CJK)


def load_vocab(path: str | Path) -> dict[str, int]:
    """vocab.txt: one token per line, its id the line number."""
    with open(path, encoding="utf-8") as f:
        return {line.rstrip("\n"): i for i, line in enumerate(f)}


def basic_tokenize(text: str) -> list[str]:
    """Cleaning, CJK isolation, whitespace split, lower case, accent stripping and punctuation split."""
    out = []
    for ch in text:
        if ch in ("\x00", "\ufffd") or _is_control(ch):
            continue
        if _is_cjk(ch):
            out.append(f" {ch} ")
        else:
            out.append(" " if _is_whitespace(ch) else ch)
    words = []
    for word in "".join(out).split():
        word = "".join(c for c in unicodedata.normalize("NFD", word.lower()) if unicodedata.category(c) != "Mn")
        cur: list[str] = []
        for ch in word:
            if _is_punctuation(ch):
                if cur:
                    words.append("".join(cur))
                    cur = []
                words.append(ch)
            else:
                cur.append(ch)
        if cur:
            words.append("".join(cur))
    return words


def wordpiece(word: str, vocab: dict[str, int], unk: str = "[UNK]") -> list[str]:
    """Greedy longest-match-first split of one word; [UNK] when too long or when some position has no match."""
    if len(word) > MAX_WORD_CHARS:
        return [unk]
    pieces, start = [], 0
    while start < len(word):
        for end in range(len(word), start, -1):
            sub = word[start:end] if start == 0 else "##" + word[start:end]
            if sub in vocab:
                pieces.append(sub)
                start = end
                break
        else:
            return [unk]
    return pieces


class BertTokenizer:
    """Lower-casing WordPiece tokenizer over a BERT vocab.txt."""

    def __init__(self, vocab: dict[str, int]) -> None:
        missing = [t for t in SPECIAL_TOKENS if t not in vocab]
        if missing:
            msg = f"vocab lacks the special tokens {missing}"
            raise ValueError(msg)
        self.vocab = vocab
        self.cls_id, self.sep_id, self.pad_id, self.unk_id = (vocab[t] for t in ("[CLS]", "[SEP]", "[PAD]", "[UNK]"))

    @classmethod
    def from_file(cls, path: str | Path) -> BertTokenizer:
        return cls(load_vocab(path))

    def tokenize(self, text: str) -> list[str]:
        out: list[str] = []
        for part in _SPECIAL_RE.split(text):
            if part in SPECIAL_TOKENS:
                out.append(part)
            elif part:
                for word in basic_tokenize(part):
                    out += wordpiece(word, self.vocab)
        return out

    def ids(self, text: str) -> list[int]:
        """Token ids of `text` without [CLS] / [SEP]."""
        return [self.vocab.get(t, self.unk_id) for t in self.tokenize(text)]

    def __call__(self, texts: list[str], max_len: int = 40) -> tuple[np.ndarray, np.ndarray]:
        """texts -> (int32 ids [n][max_len], int32 lengths [n]): [CLS] + pieces[:max_len - 2] + [SEP], [PAD] to max_len."""
        if max_len < 2:
            msg = f"max_len {max_len} leaves no room for [CLS] and [SEP]"
            raise ValueError(msg)
        ids = np.full((len(texts), max_len), self.pad_id, dtype=np.int32)
        lengths = np.empty(len(texts), dtype=np.int32)
        for i, text in enumerate(texts):
            seq = [self.cls_id, *self.ids(text)[: max_len - 2], self.sep_id]
            ids[i, : len(seq)] = seq
            lengths[i] = len(seq)
        return ids, lengths
