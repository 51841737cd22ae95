#!/usr/bin/env python
"""Generates tests/golden/clip_hard_golden.npz: HF ``transformers.CLIPVisionModelWithProjection``, fp32 on CPU, then L2
normalisation, on the "hard" weight style of oracle/clip_ref.make_weights (massive residual channels on the class token and
two patch tokens, an attention sink, peaked attention, LayerNorm gains ~2.5) and seeded pixels.  These vectors pin the fp64
oracle on those statistics and, through it, the CUDA path (tests/test_gpu_pre_ln_chain.py).

    python tests/golden/make_clip_hard_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import clip_ref as C  # noqa: E402

CASES = {
    # name: (layers, weight seed, n images, pixel seed)
    "VH2": (2, 1, 3, 4),
    "VH12": (12, 5, 4, 6),
}


def case_inputs(name):
    layers, wseed, n, pseed = CASES[name]
    g = C.VitGeometry(layers=layers)
    return g, C.make_weights(g, wseed, "hard"), C.synth_pixels(n, g, pseed)


def main():
    out = {}
    for name in CASES:
        g, flat, px = case_inputs(name)
        emb = C.forward_hf(C.build_hf_model(flat, g), px)
        out[f"{name}_emb"] = emb
        out[f"{name}_digest"] = np.frombuffer(hashlib.sha256(C.pack_blob(flat, g).tobytes()).digest(), np.uint8)
        out[f"{name}_px_sum"] = np.array([float(px.astype(np.float64).sum())])
        print(name, emb.shape, float(C.rel_l2(emb, C.forward_np(flat, px, g)).max()))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "clip_hard_golden.npz"), **out)


if __name__ == "__main__":
    main()
