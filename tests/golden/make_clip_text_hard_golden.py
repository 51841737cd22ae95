#!/usr/bin/env python
"""Generates tests/golden/clip_text_hard_golden.npz: HF ``transformers.CLIPTextModelWithProjection``, fp32 on CPU, then L2
normalisation, on the "hard" weight style of tests/clip_text_refs.make_weights (massive residual channels on position 0, an
attention sink on key 0, peaked attention, LayerNorm gains ~2.5) and seeded token ids.  These vectors pin the fp64 oracle on
those statistics and, through it, the CUDA path (tests/test_gpu_pre_ln_chain.py).

    python tests/golden/make_clip_text_hard_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "modal-examples_b200"), os.path.join(ROOT, "tests")]
import clip_text_refs as T  # noqa: E402

CASES = {
    # name: (layers, weight seed, eos_id, lens, eos padding inside len; -1: no special token, words only)
    "HA": (2, 1, 2, [77, 3, 64, 30, 2], 0),                  # ragged, EOS at len - 1
    "HB": (12, 2, 2, [2, 9, 33, 64, 65, 77], 0),             # ragged 2-77
    "HC": (12, 3, 49407, [5, 12, 40, 77], 5),               # first-match rule, 49407 padding after EOS inside len
    "HD": (2, 4, 49407, [6, 30, 77], -1),                    # no EOS: first-match pools row 0, the massive one
}


def case_inputs(name):
    layers, wseed, eos_id, lens, pad = CASES[name]
    g = T.geometry(layers=layers, eos_id=eos_id)
    ids = T.synth_ids(lens, max(lens), seed=wseed + 20, eos_pad=max(pad, 0))
    if pad < 0:
        ids = np.where(ids >= T.BOS, 1234, ids).astype(np.int32)
    return g, T.make_weights(g, wseed, "hard"), ids, np.array(lens, np.int32)


def main():
    out = {}
    for name in CASES:
        g, flat, ids, lens = case_inputs(name)
        emb = T.forward_hf(T.build_hf_model(flat, g), ids, lens)
        out[f"{name}_emb"] = emb
        out[f"{name}_ids"] = ids
        out[f"{name}_lens"] = lens
        out[f"{name}_digest"] = np.frombuffer(hashlib.sha256(T.pack_blob(flat, g).tobytes()).digest(), np.uint8)
        print(name, emb.shape, float(T.rel_l2(emb, T.forward_np(flat, ids, lens, g)).max()))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "clip_text_hard_golden.npz"), **out)


if __name__ == "__main__":
    main()
