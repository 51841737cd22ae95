"""CLIP's byte-level BPE tokeniser (``vocab.json`` + ``merges.txt``), restated from the published algorithm that
``transformers.CLIPTokenizerFast`` runs -- what infinity's ``AutoProcessor`` loads for ``openai/clip-vit-base-patch16``
(tests/test_clip_text.py checks this file against it on the same vocabulary):

* split out the literal special tokens ``<|startoftext|>`` / ``<|endoftext|>`` (case-sensitive, before normalisation), which
  map straight to their ids, as the fast tokenizer's added tokens do;
* normalise the text between them: NFC, every whitespace run -> one space, lower-case;
* pre-tokenise with CLIP's regex (contractions, letter runs, single digits, punctuation runs; whitespace dropped);
* map each piece's UTF-8 bytes to GPT-2's printable byte alphabet, BPE it with ``</w>`` marking the word end;
* ``<|startoftext|>`` ... ``<|endoftext|>``, truncated to 77 tokens with the end token kept.

Without a vocabulary offline the tokeniser falls back to CLIP's merge-free base vocabulary: the 256 byte symbols at ids
0-255, their ``</w>`` forms at 256-511 (their ids in the real vocabulary too) and the two special tokens at 49406 / 49407.
Every word then becomes one token per byte, so embeddings of strings are not the real model's -- the engine says so loudly.
"""
from __future__ import annotations

import json
import os
import unicodedata

import regex

CONTEXT_LENGTH = 77
BOS_TOKEN, EOS_TOKEN = "<|startoftext|>", "<|endoftext|>"
BASE_BOS_ID, BASE_EOS_ID = 49406, 49407
_MAX_MERGES = 49152 - 256 - 2  # the merges CLIP's tokenizer reads (the rest of merges.txt is never used)
_CACHE_MAX = 1 << 16  # words whose BPE is remembered; the cache starts over when full (a long-running server sees open-ended text)

_SPECIAL = regex.compile(r"(<\|startoftext\|>|<\|endoftext\|>)")
_PAT = regex.compile(r"""'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""", regex.IGNORECASE)
_WS = regex.compile(r"\s+")


def bytes_to_unicode() -> dict:
    """GPT-2's reversible byte -> printable character map (printable Latin-1 bytes map to themselves, the rest to 256+)."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, map(chr, cs)))


def base_vocab() -> dict:
    """CLIP's vocabulary without merges: byte symbols, their word-final forms, the two special tokens."""
    syms = list(bytes_to_unicode().values())
    vocab = {s: i for i, s in enumerate(syms + [s + "</w>" for s in syms])}
    vocab[BOS_TOKEN], vocab[EOS_TOKEN] = BASE_BOS_ID, BASE_EOS_ID
    return vocab


class ClipTokenizer:
    def __init__(self, vocab: dict | None = None, merges: list | None = None):
        self.vocab = vocab if vocab is not None else base_vocab()
        self.ranks = {tuple(m): i for i, m in enumerate(merges or [])}
        self.bos_id, self.eos_id = self.vocab[BOS_TOKEN], self.vocab[EOS_TOKEN]
        self.synthetic = vocab is None
        self._byte = bytes_to_unicode()
        self._cache: dict[str, list[int]] = {}

    @classmethod
    def from_files(cls, vocab_json: str, merges_txt: str) -> "ClipTokenizer":
        with open(vocab_json, encoding="utf-8") as f:
            vocab = json.load(f)
        with open(merges_txt, encoding="utf-8") as f:
            lines = f.read().strip().split("\n")
        if lines and lines[0].startswith("#version"):
            lines = lines[1:]
        merges = [tuple(l.split()) for l in lines[:_MAX_MERGES] if l.strip()]
        return cls(vocab, merges)

    @classmethod
    def from_dir(cls, path: str | None) -> "ClipTokenizer":
        """``vocab.json`` + ``merges.txt`` of a CLIP snapshot directory; the merge-free base vocabulary when absent."""
        if path:
            v, m = os.path.join(path, "vocab.json"), os.path.join(path, "merges.txt")
            if os.path.exists(v) and os.path.exists(m):
                return cls.from_files(v, m)
        return cls()

    def _bpe(self, piece: str) -> list[int]:
        got = self._cache.get(piece)
        if got is not None:
            return got
        word = list(piece[:-1]) + [piece[-1] + "</w>"]
        while len(word) > 1:
            best, bi = None, -1
            for i in range(len(word) - 1):
                r = self.ranks.get((word[i], word[i + 1]))
                if r is not None and (best is None or r < best):
                    best, bi = r, i
            if best is None:
                break
            a, b = word[bi], word[bi + 1]
            out, i = [], 0
            while i < len(word):  # merge every occurrence of the pair, left to right
                if i < len(word) - 1 and word[i] == a and word[i + 1] == b:
                    out.append(a + b)
                    i += 2
                else:
                    out.append(word[i])
                    i += 1
            word = out
        ids = [self.vocab[w] for w in word]
        if len(self._cache) >= _CACHE_MAX:
            self._cache.clear()
        self._cache[piece] = ids
        return ids

    def encode(self, text: str) -> list[int]:
        """Token ids of one string, ``<|startoftext|>`` and ``<|endoftext|>`` included, at most 77."""
        ids = []
        for k, part in enumerate(_SPECIAL.split(text)):
            if k % 2:  # a literal special token
                ids.append(self.vocab[part])
                continue
            for piece in _PAT.findall(_WS.sub(" ", unicodedata.normalize("NFC", part)).lower()):
                ids += self._bpe("".join(self._byte[b] for b in piece.encode("utf-8")))
        return [self.bos_id] + ids[:CONTEXT_LENGTH - 2] + [self.eos_id]

    def batch(self, texts) -> tuple:
        """(ids int32 [n, longest], lens int32 [n]): padded to the longest item with ``<|endoftext|>``, as the HF tokenizer
        pads with ``padding=True``.  Positions past lens[i] are padding."""
        import numpy as np

        enc = [self.encode(t) for t in texts]
        S = max(len(e) for e in enc)
        ids = np.full((len(enc), S), self.eos_id, np.int32)
        for i, e in enumerate(enc):
            ids[i, :len(e)] = e
        return ids, np.array([len(e) for e in enc], np.int32)
