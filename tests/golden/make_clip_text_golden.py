#!/usr/bin/env python
"""Generates tests/golden/clip_text_golden.npz by running the Python reference library -- Hugging Face
``transformers.CLIPTextModelWithProjection`` (the text tower of the reference's ``openai/clip-vit-base-patch16``,
``06_gpu_and_ml/embeddings/image_embeddings_infinity.py:76-77``) -- on seeded weights and seeded token ids, fp32 on CPU,
followed by L2 normalisation.  These vectors pin the numpy restatement (tests/clip_text_refs.py) and, through it, the CUDA path.

    python tests/golden/make_clip_text_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "modal-examples_b200"), os.path.join(ROOT, "tests")]
import clip_text_refs as T  # noqa: E402

CASES = {
    # name: (layers, style, weight seed, eos_id, lens, eos padding inside len)
    "TA": (2, "trained", 1, 2, [5, 17, 2, 77], 0),                                    # EOS at len - 1
    "TB": (12, "hf", 0, 2, [2, 9, 33, 64, 65, 77], 0),                                # ragged 2-77, EOS at len - 1
    "TC": (12, "trained", 2, 2, [12, 40, 77], 5),                                     # 49407 padding after EOS inside len
    "TD": (2, "trained", 3, 2, [6, 30, 77], -1),                                      # no EOS, legacy argmax branch
    "TE": (2, "trained", 3, 49407, [6, 30, 77], -1),                                  # no EOS, first-match branch: row 0
}


def case_inputs(name):
    layers, style, wseed, eos_id, lens, pad = CASES[name]
    g = T.geometry(layers=layers, eos_id=eos_id)
    S = max(lens)
    ids = T.synth_ids(lens, S, seed=wseed + 10, eos_pad=max(pad, 0))
    if pad < 0:  # no special token anywhere, words only: the legacy branch pools the largest word id, first-match row 0
        ids = np.where(ids >= T.BOS, 1234, ids).astype(np.int32)
    return g, T.make_weights(g, wseed, style), ids, np.array(lens, np.int32)


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
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "clip_text_golden.npz"), **out)


if __name__ == "__main__":
    main()
