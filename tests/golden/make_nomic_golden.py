#!/usr/bin/env python
"""Generates tests/golden/nomic_golden.npz: nomic-bert encoders run through Hugging Face ``transformers.NomicBertModel`` fp32
on CPU (sdpa attention) with seeded weights (tests/nomic_refs.py), mean- and CLS-pooled and L2-normalised, items one at a time
and unpadded.

  * ``l12_hf`` / ``l12_trained``: 12 layers, max_position_embeddings 2048, lengths L12 (ragged, up to 2048);
  * ``l2_hf_8k`` / ``l2_trained_8k``: 2 layers, max_position_embeddings 8192, lengths L8K (up to 8192).

For each case ``<case>_ids`` int32 [items, max len] (zero-padded), ``<case>_lens``, ``<case>_mean`` / ``<case>_cls`` float32
[items, 768], and the emulated fp16-operand floor of the GPU path on the same inputs, ``<case>_floor_mean`` / ``_floor_cls``
(float64 [items]: nomic_refs.emulate_forward against the fp64 oracle), which the parity bars (nomic_refs.BARS) must be at
least twice.  Only pooled vectors are kept.  The archive is written with fixed zip timestamps, so running the script again
rewrites the file byte for byte.

    python tests/golden/make_nomic_golden.py    # needs torch + transformers; ~15 min on 8 CPU cores
"""
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import nomic_refs as N  # noqa: E402

# name: (layers, max_pos, style, weight seed, lengths)
L12 = [2048, 1000, 513, 129, 1]
L8K = [8192, 4097, 1000, 513]
CASES = {
    "l12_hf": (12, 2048, "hf", 51, L12),
    "l12_trained": (12, 2048, "trained", 52, L12),
    "l2_hf_8k": (2, 8192, "hf", 53, L8K),
    "l2_trained_8k": (2, 8192, "trained", 54, L8K),
}
INPUT_SEED = 55


def case_inputs(name):
    layers, max_pos, style, seed, lens = CASES[name]
    g = N.geometry(layers=layers, max_pos=max_pos)
    rng = np.random.default_rng(INPUT_SEED + list(CASES).index(name))
    ids = np.zeros((len(lens), max(lens)), np.int32)
    for i, n in enumerate(lens):
        ids[i, :n] = rng.integers(1000, g["vocab"], n)
    return g, N.make_weights(g, seed, style), ids, np.array(lens, np.int32)


def save(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)


def main():
    import torch

    torch.manual_seed(0)
    out = {}
    for name in CASES:
        g, flat, ids, lens = case_inputs(name)
        hf = N.hidden_hf(N.build_hf_model(flat, g, attn="sdpa"), ids, lens)
        ref = N.hidden_np(flat, ids, lens, g)
        emu = N.emulate_hidden(flat, ids, lens, g)
        out[f"{name}_ids"], out[f"{name}_lens"] = ids, lens
        for pooling in ("mean", "cls"):
            r = N.pool(ref, pooling)
            out[f"{name}_{pooling}"] = N.pool(hf, pooling).astype(np.float32)
            out[f"{name}_floor_{pooling}"] = np.linalg.norm(N.pool(emu, pooling) - r, axis=-1) / np.linalg.norm(r, axis=-1)
            print(name, pooling, "HF vs fp64 oracle", (np.linalg.norm(out[f"{name}_{pooling}"] - r, axis=-1)).max(),
                  "floor", out[f"{name}_floor_{pooling}"].max(), flush=True)
    save(os.path.join(HERE, "nomic_golden.npz"), out)


if __name__ == "__main__":
    main()
