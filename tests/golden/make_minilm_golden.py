#!/usr/bin/env python
"""Generates tests/golden/minilm_golden.npz: the all-MiniLM-L6-v2 geometry (sentence-transformers/all-MiniLM-L6-v2: hidden
384, 12 heads of 32, inter 1536, 6 layers -- bge-small's geometry with 6 layers) run through Hugging Face
``transformers.BertModel`` fp32 on CPU with seeded weights, then sentence-transformers' mean pooling over the valid tokens
and L2 normalisation (tests/mean_pool_refs.py: forward_hf_mean).  Ragged lengths, including one-token items.

    python tests/golden/make_minilm_golden.py    # rewrites minilm_golden.npz (needs torch + transformers)
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
from make_golden import blob_digest  # noqa: E402
import mean_pool_refs as MP  # noqa: E402

MINILM = dict(hidden=384, heads=12, inter=1536, layers=6)

CASES = {
    # name: (style, weight seed, input spec); specs: ("ragged", n, max_len, seed, min_len) as in make_golden.py, or
    # ("lens", [lengths], max_len, seed): synth_ragged's ids with the given lengths
    "A": ("hf", 0, ("ragged", 5, 96, 1, 1)),
    "B": ("hf", 0, ("lens", [1, 2, 1, 37, 128, 1], 128, 7)),
    "C": ("trained", 3, ("ragged", 6, 200, 5, 1)),
    "D": ("trained", 3, ("lens", [1, 512, 3, 1, 300], 512, 8)),
}


def geometry():
    return R.BertGeometry(**MINILM)


def case_inputs(spec):
    if spec[0] == "ragged":
        _, n, s, seed, min_len = spec
        return R.synth_ragged(n, s, seed=seed, min_len=min_len)
    _, lens, s, seed = spec
    ids, _ = R.synth_ragged(len(lens), s, seed=seed, min_len=s)
    lens = np.asarray(lens, np.int32)
    for i, n in enumerate(lens):
        ids[i, n:] = 0
        if n > 1:
            ids[i, n - 1] = 102
    return ids, lens


def main():
    g = geometry()
    out = {}
    cache = {}
    for name, (style, wseed, spec) in CASES.items():
        key = (style, wseed)
        if key not in cache:
            flat = R.make_weights(g, wseed, style)
            cache[key] = (flat, R.build_hf_model(flat, g), blob_digest(flat, g))
        flat, model, digest = cache[key]
        ids, lens = case_inputs(spec)
        emb = MP.forward_hf_mean(model, ids, lens)
        out[f"{name}_emb"] = emb
        out[f"{name}_digest"] = np.frombuffer(bytes.fromhex(digest), np.uint8)
        out[f"{name}_ids_sum"] = np.array([int(ids.astype(np.int64).sum())])
        print(name, emb.shape, digest[:16], float(np.linalg.norm(emb, axis=1).mean()))
    np.savez_compressed(os.path.join(HERE, "minilm_golden.npz"), **out)


if __name__ == "__main__":
    main()
