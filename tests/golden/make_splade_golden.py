#!/usr/bin/env python
"""Generates tests/golden/splade_golden.npz: SPLADE sparse encoders run through Hugging Face ``transformers.BertForMaskedLM``
fp32 on CPU with seeded weights (tests/splade_refs.py), pooled as sentence-transformers' ``SpladePooling(max, relu)`` pools
them, on one ragged batch.

  * bge-base geometry (naver/splade-v3's), 2 and 12 layers, weight styles `hf` (dense: nearly every word non-zero) and
    `splade` (50-400 non-zero words per 64-256-token item);
  * bge-small geometry, 2 layers, `splade`.

The batch spans the 64-token buckets 64 .. 512 and holds an item of one token and items of 64k - 1 and 64k + 1 tokens.  A
`splade` case's [items, vocab] output is stored whole, as CSR of its non-zeros (`<case>_indptr`, `_indices` uint16, `_values`).
An `hf` case is dense -- nearly every word non-zero -- and is stored at the fixed word sample HF_COLS only (`<case>_values`
[items, len(HF_COLS)]): 512 seeded words plus the vocabulary's last 32, which lie in the decoder's last, partly padded
column tile.  That keeps the file under 100 KB.  Running the script again rewrites the file byte for byte.

    python tests/golden/make_splade_golden.py    # needs torch + transformers
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import bge_ref as R  # noqa: E402
import splade_refs as SR  # noqa: E402

SMALL = dict(hidden=384, heads=12, inter=1536)
# name: (geometry kwargs, layers, style, weight seed)
CASES = {
    "base2_hf": ({}, 2, "hf", 41),
    "base2_splade": ({}, 2, "splade", 41),
    "base12_hf": ({}, 12, "hf", 42),
    "base12_splade": ({}, 12, "splade", 42),
    "small2_splade": (SMALL, 2, "splade", 43),
}
LENS = [1, 63, 64, 65, 127, 129, 300, 512]
INPUT_SEED = 44
VOCAB = 30522
HF_COLS = np.union1d(np.random.default_rng(45).choice(VOCAB - 32, 512, replace=False), np.arange(VOCAB - 32, VOCAB))


def geometry(name):
    kw, layers, _, _ = CASES[name]
    return R.BertGeometry(layers=layers, **kw)


def weights(name):
    _, _, style, seed = CASES[name]
    return SR.make_splade_weights(geometry(name), seed, style)


def inputs():
    """ids [8, 512]: [CLS] ... [SEP] within each length, interior ids uniform in [1000, 30522), [PAD] after it."""
    rng = np.random.default_rng(INPUT_SEED)
    ids = np.zeros((len(LENS), max(LENS)), np.int32)
    for i, n in enumerate(LENS):
        ids[i, :n] = rng.integers(1000, 30522, size=n)
        ids[i, 0] = 101
        if n > 1:
            ids[i, n - 1] = 102
    return ids, np.asarray(LENS, np.int32)


def reference(golden, name):
    """(cols, values [items, len(cols)] float32): the words a case stores and HF's values there -- every word of a `splade`
    case (from its CSR), HF_COLS of an `hf` case."""
    if CASES[name][2] == "hf":
        return HF_COLS, golden[f"{name}_values"]
    ptr, idx, val = golden[f"{name}_indptr"], golden[f"{name}_indices"].astype(np.int64), golden[f"{name}_values"]
    out = np.zeros((len(ptr) - 1, VOCAB), np.float32)
    for i in range(len(ptr) - 1):
        out[i, idx[ptr[i]:ptr[i + 1]]] = val[ptr[i]:ptr[i + 1]]
    return np.arange(VOCAB), out


def main():
    ids, lens = inputs()
    out = {"ids": ids, "lens": lens}
    for name in CASES:
        g, flat = geometry(name), weights(name)
        v = SR.splade_hf(SR.build_hf_masked_lm(flat, g), ids, lens)
        nz = v > 0
        if CASES[name][2] == "hf":
            out[f"{name}_values"] = v[:, HF_COLS].astype(np.float32)
        else:
            out[f"{name}_indptr"] = np.concatenate([[0], np.cumsum(nz.sum(1))]).astype(np.int32)
            out[f"{name}_indices"] = np.nonzero(nz)[1].astype(np.uint16)
            out[f"{name}_values"] = v[nz].astype(np.float32)
        print(name, "non-zero words per item", nz.sum(1).tolist(), "max", float(v.max()))
    np.savez_compressed(os.path.join(HERE, "splade_golden.npz"), **out)


if __name__ == "__main__":
    main()
