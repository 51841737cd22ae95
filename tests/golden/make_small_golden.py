#!/usr/bin/env python
"""Generates tests/golden/bge_small_golden.npz: the bge-small geometry (hidden 384, 12 heads of 32, inter 1536 --
BAAI/bge-small-en-v1.5, the model the reference's Wikipedia embedding example serves) run through Hugging Face
``transformers.BertModel`` fp32 on CPU with seeded weights, then CLS pooling and L2 normalisation, exactly as
make_golden.py does for bge-base.

    python tests/golden/make_small_golden.py    # rewrites bge_small_golden.npz (needs torch + transformers)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import bge_ref as R  # noqa: E402
from make_golden import blob_digest, case_inputs  # noqa: E402

SMALL = dict(hidden=384, heads=12, inter=1536)

CASES = {
    # name: (layers, style, weight seed, input spec) -- input specs as in make_golden.py
    "A": (12, "hf", 0, ("full", 2, 512, 0)),
    "B": (12, "hf", 0, ("ragged", 5, 96, 1, 1)),
    "C": (2, "trained", 3, ("ragged", 3, 200, 5, 3)),
    "D": (12, "trained", 0, ("ragged", 4, 512, 1, 16)),
    "E": (12, "hard", 0, ("ragged", 4, 512, 2, 64)),
}


def geometry(layers):
    return R.BertGeometry(layers=layers, **SMALL)


def main():
    out = {}
    cache = {}
    for name, (layers, style, wseed, spec) in CASES.items():
        g = geometry(layers)
        key = (layers, style, wseed)
        if key not in cache:
            flat = R.make_weights(g, wseed, style)
            cache[key] = (flat, R.build_hf_model(flat, g), blob_digest(flat, g))
        flat, model, digest = cache[key]
        ids, lens = case_inputs(spec)
        emb = R.forward_hf(model, ids, lens)
        out[f"{name}_emb"] = emb
        out[f"{name}_digest"] = np.frombuffer(bytes.fromhex(digest), np.uint8)
        out[f"{name}_ids_sum"] = np.array([int(ids.astype(np.int64).sum())])
        print(name, emb.shape, digest[:16], float(np.linalg.norm(emb, axis=1).mean()))
    np.savez_compressed(os.path.join(HERE, "bge_small_golden.npz"), **out)


if __name__ == "__main__":
    main()
