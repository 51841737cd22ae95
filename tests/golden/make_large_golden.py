#!/usr/bin/env python
"""Generates tests/golden/bge_large_golden.npz: the bge-large geometry (hidden 1024, 16 heads of 64, inter 4096 --
BAAI/bge-large-en-v1.5, BERT-large; also the shape of e5-large-v2, gte-large and mxbai-embed-large-v1) run through Hugging
Face ``transformers.BertModel`` fp32 on CPU with seeded weights, then CLS pooling and L2 normalisation as make_golden.py does
for bge-base -- or, for the mean-pooled case, sentence-transformers' mean over the valid tokens (tests/mean_pool_refs.py).

The ``hard`` weight style appears at 2 layers only: at this width it drives a deep stack far enough from fp64 that even HF
fp32 disagrees with the fp64 oracle by 1.3e-4 (12 layers) and 8.8e-3 (24 layers) -- see DESIGN.md section 2.

    python tests/golden/make_large_golden.py    # rewrites bge_large_golden.npz (needs torch + transformers, ~3 GB of RAM)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from oracle import bge_ref as R  # noqa: E402
from make_golden import blob_digest, case_inputs  # noqa: E402
import mean_pool_refs as MP  # noqa: E402

LARGE = dict(hidden=1024, heads=16, inter=4096)

CASES = {
    # name: (layers, style, weight seed, input spec, pooling) -- input specs as in make_golden.py
    "A": (24, "hf", 0, ("full", 2, 512, 0), "cls"),
    "B": (24, "trained", 0, ("ragged", 4, 512, 1, 16), "cls"),
    "C": (2, "trained", 3, ("ragged", 3, 200, 5, 3), "cls"),
    "D": (2, "hard", 0, ("ragged", 4, 512, 2, 64), "cls"),
    "E": (24, "trained", 0, ("ragged", 5, 300, 4, 1), "mean"),
}


def geometry(layers):
    return R.BertGeometry(layers=layers, **LARGE)


def main():
    out = {}
    cache = {}
    for name, (layers, style, wseed, spec, pooling) in CASES.items():
        g = geometry(layers)
        key = (layers, style, wseed)
        if key not in cache:
            cache.clear()  # one 24-layer model in memory at a time
            flat = R.make_weights(g, wseed, style)
            cache[key] = (flat, R.build_hf_model(flat, g), blob_digest(flat, g))
        flat, model, digest = cache[key]
        ids, lens = case_inputs(spec)
        emb = MP.forward_hf_mean(model, ids, lens) if pooling == "mean" else R.forward_hf(model, ids, lens)
        out[f"{name}_emb"] = emb
        out[f"{name}_digest"] = np.frombuffer(bytes.fromhex(digest), np.uint8)
        out[f"{name}_ids_sum"] = np.array([int(ids.astype(np.int64).sum())])
        print(name, emb.shape, digest[:16], float(np.linalg.norm(emb, axis=1).mean()))
    np.savez_compressed(os.path.join(HERE, "bge_large_golden.npz"), **out)


if __name__ == "__main__":
    main()
