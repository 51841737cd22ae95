#!/usr/bin/env python
"""Diagnostics: is an item's result bit-identical whatever batch it travels in?  Kernel by kernel."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "modal-examples_b200"))
import numpy as np
import b200rt
from oracle import bge_ref as R

b200rt.init(1)
g = R.BertGeometry(layers=2)
flat = R.make_weights(g, 3, "trained")
model = b200rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g))
n, S = 45, 256
ids, lens = R.synth_ragged(n, S, seed=11, min_len=2)
for L in (0, 1, 2):
    full = model.debug_residual(ids, lens, L)
    part = np.concatenate([model.debug_residual(ids[i:i + 32], lens[i:i + 32], L) for i in range(0, n, 32)])
    d = full != part
    # only rows < len matter
    valid = np.arange(S)[None, :] < lens[:, None]
    dv = d & valid[:, :, None]
    print(f"residual stream after {L} layers: {int(dv.sum())} differing valid elements of {int(valid.sum()) * 768}; items affected {sorted(set(np.where(dv.any((1, 2)))[0].tolist()))[:20]}")
    if dv.any():
        it = np.where(dv.any((1, 2)))[0][0]
        rows = np.where(dv[it].any(1))[0]
        cols = np.where(dv[it].any(0))[0]
        print(f"   item {it} (len {lens[it]}): rows {rows[:10]}.. ({len(rows)}), cols {cols[:10]}.. ({len(cols)}), max abs diff {np.abs(full - part)[dv].max():.3e}")
# attention alone
rng = np.random.default_rng(0)
qkv = rng.standard_normal((n * S, 2304)).astype(np.float16)
full, _ = b200rt.debug_attention(qkv, lens, n, S)
part = np.concatenate([b200rt.debug_attention(qkv[i * S:(i + 32) * S], lens[i:i + 32], min(32, n - i), S)[0] for i in range(0, n, 32)])
valid = (np.arange(S)[None, :] < lens[:, None]).reshape(-1)
d = (full != part) & valid[:, None]
print("attention alone: differing valid elements", int(d.sum()))
# gemm epi 2 alone with LN: rows of a big batch vs the same rows in a small batch
M, K, N = 45 * 256, 768, 768
a = rng.standard_normal((M, K)).astype(np.float16)
w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
bias = rng.standard_normal(N).astype(np.float32)
resid = rng.standard_normal((M, N)).astype(np.float32)
def partials(y):
    sl = y.astype(np.float64).reshape(y.shape[0], -1, 128)
    return np.stack([sl.sum(-1), ((sl - sl.mean(-1, keepdims=True)) ** 2).sum(-1)], -1).astype(np.float32)
gam = (1 + 0.1 * rng.standard_normal(N)).astype(np.float32); bet = (0.1 * rng.standard_normal(N)).astype(np.float32)
for epi in (0, 2):
    kw = dict(ln_stats=partials(resid if epi == 2 else a.astype(np.float32)))
    if epi == 2:
        kw.update(ln_gamma=gam, ln_beta=bet)
    o_full = b200rt.debug_gemm(epi, a, w, bias, resid if epi == 2 else None, **kw)[0]
    m0 = 32 * 256
    kw2 = {k: (v[:m0] if k == "ln_stats" else v) for k, v in kw.items()}
    o_part = b200rt.debug_gemm(epi, a[:m0], w, bias, resid[:m0] if epi == 2 else None, **kw2)[0]
    print(f"gemm epi {epi}: differing elements in the first {m0} rows: {int((o_full[:m0] != o_part).sum())}")
b200rt.shutdown()
