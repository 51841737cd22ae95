#!/usr/bin/env python
"""Generates tests/golden/rerank_golden.npz: BERT cross-encoders / sequence classifiers run through Hugging Face
``transformers.BertForSequenceClassification`` fp32 on CPU with seeded weights (tests/rerank_refs.py), on ragged batches of
sentence pairs: [CLS] a [SEP] b [SEP] with token type 1 on b, plus single sequences.

  * reranker cases: cross-encoder/ms-marco-MiniLM-L-6-v2's geometry (hidden 384, 12 heads of 32, inter 1536), one label,
    6 and 12 layers (-L-6-v2 / -L-12-v2), weight styles `hf` and `trained`;
  * a bge-base-geometry classifier with two labels and 2 layers (`trained`).

The batch spans the 64-token buckets 64 .. 256 and holds a second segment of one token ([SEP] alone), an empty first text,
single sequences (segs == lens) and an item of one token.  Running the script again rewrites the file byte for byte.

    python tests/golden/make_rerank_golden.py    # needs torch + transformers
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import bge_ref as R  # noqa: E402
import rerank_refs as RR  # noqa: E402

MINILM = dict(hidden=384, heads=12, inter=1536)
# name: (geometry kwargs, layers, style, weight seed, num_labels)
CASES = {
    "l6_hf": (MINILM, 6, "hf", 11, 1),
    "l6_trained": (MINILM, 6, "trained", 11, 1),
    "l12_hf": (MINILM, 12, "hf", 12, 1),
    "l12_trained": (MINILM, 12, "trained", 12, 1),
    "base2_trained": ({}, 2, "trained", 13, 2),
}
S = 200
LENS = [200, 3, 64, 65, 130, 128, 129, 17, 96, 190, 40, 1]
SEGS = [120, 2, 63, 65, 30, 128, 100, 16, 48, 11, 40, 1]
INPUT_SEED = 21


def geometry(name):
    kw, layers, _, _, _ = CASES[name]
    return R.BertGeometry(layers=layers, **kw)


def weights(name):
    _, _, style, seed, L = CASES[name]
    return RR.make_classifier_weights(geometry(name), seed, style, L)


def inputs():
    return RR.synth_pairs(LENS, SEGS, S, INPUT_SEED)


def main():
    ids, lens, segs = inputs()
    out = {"ids": ids, "lens": lens, "segs": segs}
    for name in CASES:
        g, flat = geometry(name), weights(name)
        logits = RR.classify_hf(RR.build_hf_classifier(flat, g), ids, lens, segs)
        out[f"{name}_logits"] = logits
        print(name, logits.shape, float(logits.min()), float(logits.max()))
    path = os.path.join(HERE, "rerank_golden.npz")
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    main()
