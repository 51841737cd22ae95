"""BERT uncased tokenisation (BasicTokenizer + greedy WordPiece), restated from the published algorithm that
``transformers.BertTokenizer`` implements (tests/test_tokenizer.py checks this file against it on the same
vocabulary).  TEI tokenises with the model repo's ``tokenizer.json``; no BERT vocabulary exists offline,
so a real ``vocab.txt`` is optional (``--tokenizer-vocab`` / ``B200RT_VOCAB``) and the
fallback is a deterministic SYNTHETIC vocabulary -- the server says so at start-up; embeddings of strings are
then not comparable with the real model's (token-id inputs are unaffected)."""
from __future__ import annotations

import unicodedata

PAD, UNK, CLS, SEP, MASK = 0, 100, 101, 102, 103
VOCAB_SIZE = 30522
MAX_CHARS_PER_WORD = 100  # HF WordpieceTokenizer.max_input_chars_per_word


def load_vocab(path: str) -> dict:
    vocab = {}
    with open(path, encoding="utf-8") as f:
        for i, line in enumerate(f):
            vocab[line.rstrip("\n")] = i
    return vocab


def synthetic_vocab() -> list:
    """30 522 entries with BERT's special-token ids; every printable ASCII character (bare and ##-continued) so that
    nothing maps to [UNK], then letter n-grams and digit groups so that ordinary text needs ~3 pieces per word."""
    toks = ["[PAD]"] + [f"[unused{i}]" for i in range(99)] + ["[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    seen = set(toks)

    def add(t):
        if t not in seen and len(toks) < VOCAB_SIZE:
            seen.add(t)
            toks.append(t)

    chars = [chr(c) for c in range(33, 127) if not ("A" <= chr(c) <= "Z")]
    for c in chars:
        add(c)
    for c in chars:
        add("##" + c)
    letters = "abcdefghijklmnopqrstuvwxyz"
    for a in letters:
        for b in letters:
            add(a + b)
            add("##" + a + b)
    for n in range(100):
        add(str(n))
        add("##" + str(n))
    vowels, cons = "aeiou", "bcdfghjklmnpqrstvwxyz"
    for a in cons:          # consonant-vowel-consonant trigrams, the commonest English shapes
        for b in vowels:
            for c in cons:
                add(a + b + c)
                add("##" + a + b + c)
    for a in vowels:
        for b in cons:
            for c in vowels:
                add(a + b + c)
                add("##" + a + b + c)
    i = 0
    while len(toks) < VOCAB_SIZE:  # pad deterministically
        add(f"[synthetic{i}]")
        i += 1
    return toks


def _is_whitespace(ch):
    return ch in " \t\n\r" or unicodedata.category(ch) == "Zs"


def _is_control(ch):
    if ch in "\t\n\r":
        return False
    return unicodedata.category(ch).startswith("C")


def _is_punctuation(ch):
    cp = ord(ch)
    if 33 <= cp <= 47 or 58 <= cp <= 64 or 91 <= cp <= 96 or 123 <= cp <= 126:
        return True
    return unicodedata.category(ch).startswith("P")


def _is_cjk(cp):
    return (0x4E00 <= cp <= 0x9FFF or 0x3400 <= cp <= 0x4DBF or 0x20000 <= cp <= 0x2A6DF or 0x2A700 <= cp <= 0x2B73F or
            0x2B740 <= cp <= 0x2B81F or 0x2B820 <= cp <= 0x2CEAF or 0xF900 <= cp <= 0xFAFF or 0x2F800 <= cp <= 0x2FA1F)


def basic_tokenize(text: str) -> list:
    """Clean, pad CJK, lower-case + strip accents, split on whitespace and punctuation."""
    out = []
    for ch in text:
        cp = ord(ch)
        if cp == 0 or cp == 0xFFFD or _is_control(ch):
            continue
        if _is_whitespace(ch):
            out.append(" ")
        elif _is_cjk(cp):
            out.extend((" ", ch, " "))
        else:
            out.append(ch)
    text = unicodedata.normalize("NFC", "".join(out))
    words = []
    for tok in text.split():
        tok = tok.lower()
        tok = "".join(c for c in unicodedata.normalize("NFD", tok) if unicodedata.category(c) != "Mn")
        cur = []
        for ch in tok:
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


class WordPiece:
    def __init__(self, vocab=None):
        if vocab is None:
            vocab = {t: i for i, t in enumerate(synthetic_vocab())}
            self.synthetic = True
        else:
            self.synthetic = False
        self.vocab = vocab
        self.unk = vocab.get("[UNK]", UNK)
        self.cls = vocab.get("[CLS]", CLS)
        self.sep = vocab.get("[SEP]", SEP)

    def word_ids(self, word: str) -> list:
        if len(word) > MAX_CHARS_PER_WORD:
            return [self.unk]
        ids, start = [], 0
        while start < len(word):
            end, cur = len(word), None
            while start < end:
                sub = word[start:end]
                if start > 0:
                    sub = "##" + sub
                if sub in self.vocab:
                    cur = self.vocab[sub]
                    break
                end -= 1
            if cur is None:
                return [self.unk]
            ids.append(cur)
            start = end
        return ids

    def encode(self, text: str, max_len: int = 512, truncate: bool = False) -> list:
        """[CLS] pieces [SEP]; raises ValueError when longer than max_len and not truncating (TEI: 413)."""
        ids = [self.cls]
        for w in basic_tokenize(text):
            ids.extend(self.word_ids(w))
        ids.append(self.sep)
        if len(ids) > max_len:
            if not truncate:
                raise ValueError(f"`inputs` must have less than {max_len} tokens. Given: {len(ids)}")
            ids = ids[: max_len - 1] + [self.sep]
        return ids

    def pieces(self, text: str) -> list:
        """The WordPiece ids of ``text``, no special tokens."""
        ids = []
        for w in basic_tokenize(text):
            ids.extend(self.word_ids(w))
        return ids

    def encode_pair(self, a: str, b: str, max_len: int = 512, truncate: bool = False) -> tuple[list, int]:
        """``[CLS] a [SEP] b [SEP]`` and where b's segment (token type 1) starts: ``(ids, seg)``.  Longer than max_len: raises
        ValueError unless truncating (TEI: 413), else trims the pair as the Rust tokenizers' ``longest_first`` strategy does
        (what TEI runs, and ``BertTokenizerFast(a, b, truncation="longest_first")``): with m = max_len - 3 tokens for the two
        texts, a shorter text that fits in half of m is kept whole and the other gets the rest; otherwise each gets m // 2 and
        the longer one (b on a tie) the odd token."""
        pa, pb = self.pieces(a), self.pieces(b)
        total = len(pa) + len(pb) + 3
        if total > max_len:
            if not truncate:
                raise ValueError(f"`inputs` must have less than {max_len} tokens. Given: {total}")
            na, nb = _longest_first(len(pa), len(pb), max(max_len - 3, 0))
            pa, pb = pa[:na], pb[:nb]
        ids = [self.cls] + pa + [self.sep] + pb + [self.sep]
        return ids, len(pa) + 2


def _longest_first(n_a: int, n_b: int, m: int) -> tuple[int, int]:
    """Lengths two texts of n_a and n_b tokens keep under the tokenizers crate's LongestFirst truncation to m tokens together."""
    swap = n_a > n_b
    n1, n2 = (n_b, n_a) if swap else (n_a, n_b)  # n1 <= n2
    if n1 > m:
        n2 = n1
    else:
        n2 = max(n1, m - n1)
    if n1 + n2 > m:
        n1 = m // 2
        n2 = n1 + m % 2
    ka, kb = (n2, n1) if swap else (n1, n2)
    return min(ka, n_a), min(kb, n_b)
