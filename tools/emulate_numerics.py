#!/usr/bin/env python
"""CPU emulation of the GPU path's numerics (diagnostics; imports the oracle, so this is a tool, not product code):
rounds to fp16 exactly where the kernels do and accumulates in fp32, to predict the parity margin of a design before it is
written as CUDA.

  mode "current": x16 = fp16(LN(y)) feeds QKV / FFN1 (round-1 design, LayerNorm kernels materialise x16)
  mode "fold"   : y16 = fp16(y) (the raw pre-LayerNorm residual) feeds QKV / FFN1 with gamma folded into the weight columns;
                  and the weight rows centred; the epilogue applies rstd * acc + (W beta + b)   (round-2 design, no LN kernels)

    python tools/emulate_numerics.py [--geometry base|small|large] [--style hf|trained|hard] [--layers 12] [--items 4] [--seq 512]
                                     [--pooling cls|mean]

--geometry small: bge-small (hidden 384, 12 heads of 32, inter 1536) instead of bge-base; --geometry large: bge-large
(hidden 1024, 16 heads of 64, inter 4096).
--pooling mean: sentence-transformers' mean of the valid tokens' final hidden states (all-MiniLM-L6-v2, e5, gte) instead of
the [CLS] row, against the fp64 oracle pooled the same way (tests/mean_pool_refs.py).
"""
import argparse
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import bge_ref as R  # noqa: E402
import mean_pool_refs as MP  # noqa: E402

GEOMETRIES = {"base": {}, "small": dict(hidden=384, heads=12, inter=1536), "large": dict(hidden=1024, heads=16, inter=4096)}

f16 = lambda a: a.astype(np.float16).astype(np.float32)  # noqa: E731


def gelu32(x):
    from scipy.special import erf

    return (x * 0.5 * (1.0 + erf(x.astype(np.float64) / math.sqrt(2.0)))).astype(np.float32)


def stats(y, eps):
    mu = y.mean(-1, keepdims=True, dtype=np.float32)
    xc = y - mu
    var = (xc * xc).mean(-1, keepdims=True, dtype=np.float32)
    return mu, (1.0 / np.sqrt(var + eps)).astype(np.float32)


def emulate(flat, ids, lens, g, mode="current", p_sum="exact", keep=(), pooling="cls"):
    """keep: names of rounding points left in fp32 (ablation): x, w, qkv, p, ctx, ffn"""
    r = lambda name, a: a if name in keep else f16(a)  # noqa: E731
    B, S = ids.shape
    h, nh, dh = g.hidden, g.heads, g.head_dim
    W = {k: v.astype(np.float32) for k, v in flat.items()}
    y = (W["emb.word"][ids] + W["emb.type"][0]) + W["emb.pos"][:S][None]
    ln = ("emb.ln.g", "emb.ln.b")
    keymask = np.arange(S)[None, :] >= np.asarray(lens)[:, None]
    k2 = np.float32(1.4426950408889634 / math.sqrt(dh))  # softmax scale 1 / sqrt(d) in base 2

    def ln_apply(y, ln):
        mu, rstd = stats(y, g.eps)
        return ((y - mu) * rstd * W[ln[0]] + W[ln[1]]).astype(np.float32)

    def gemm_after_ln(y, ln, w, b):
        if mode == "current":
            return r("x", ln_apply(y, ln)) @ r("w", W[w]).T + W[b]
        mu, rstd = stats(y, g.eps)
        wg = W[w] * W[ln[0]][None, :]
        wp = r("w", wg - wg.mean(1, keepdims=True, dtype=np.float32))  # gamma folded into the columns, rows centred, rounded once
        acc = r("x", y) @ wp.T                                         # the row mean cancels inside the GEMM
        c = W[w] @ W[ln[1]] + W[b]
        return rstd * acc + c

    for l in range(g.layers):
        p = f"l{l}."
        qkv = r("qkv", gemm_after_ln(y, ln, p + "qkv.w", p + "qkv.b"))
        q, k, v = (qkv[..., j * h:(j + 1) * h].reshape(B, S, nh, dh).transpose(0, 2, 1, 3) for j in range(3))
        s = q @ k.transpose(0, 1, 3, 2)
        s = np.where(keymask[:, None, None, :], -np.inf, s)
        m = s.max(-1, keepdims=True)
        e = np.exp2((s - m) * k2).astype(np.float32)
        e16 = r("p", e)
        lsum = (e16 if p_sum == "p16" else e).sum(-1, keepdims=True, dtype=np.float32)
        ctx = r("ctx", (e16 @ v) / lsum).transpose(0, 2, 1, 3).reshape(B, S, h)
        x = ln_apply(y, ln)
        y = ctx @ r("w", W[p + "ao.w"]).T + W[p + "ao.b"] + x
        ln = (p + "ln1.g", p + "ln1.b")
        ffn = r("ffn", gelu32(gemm_after_ln(y, ln, p + "ff1.w", p + "ff1.b")))
        x = ln_apply(y, ln)
        y = ffn @ r("w", W[p + "ff2.w"]).T + W[p + "ff2.b"] + x
        ln = (p + "ln2.g", p + "ln2.b")
    if pooling == "mean":  # fp32 LayerNorm of every valid row, fp32 masked mean
        h = ln_apply(y, ln) * (~keymask)[..., None]
        pooled = (h.sum(1, dtype=np.float32) / np.asarray(lens, np.float32)[:, None]).astype(np.float32)
    else:
        pooled = ln_apply(y[:, 0, :], ln)
    return pooled / np.maximum(np.sqrt((pooled * pooled).sum(-1, keepdims=True)), 1e-12)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--geometry", choices=tuple(GEOMETRIES), default="base")
    ap.add_argument("--style", default="hf")
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--items", type=int, default=4)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--ablate", action="store_true")
    ap.add_argument("--pooling", choices=("cls", "mean"), default="cls")
    a = ap.parse_args()
    g = R.BertGeometry(layers=a.layers, **GEOMETRIES[a.geometry])
    flat = R.make_weights(g, a.seed, a.style)
    ids, lens = R.synth_ragged(a.items, a.seq, seed=1, min_len=max(1, a.seq // 4))
    if a.pooling == "mean":
        ref = MP.forward_np_mean(flat, ids, lens, g)
        hf = MP.forward_hf_mean(R.build_hf_model(flat, g), ids, lens)
    else:
        ref = R.forward_np(flat, ids, lens, g, dtype=np.float64)
        hf = R.forward_hf(R.build_hf_model(flat, g), ids, lens)
    print(f"geometry {a.geometry} style {a.style} layers {a.layers} items {a.items} x {a.seq} pooling {a.pooling}")
    print("  HF fp32 vs numpy fp64     :", R.rel_l2(hf, ref).max())
    for mode in ("current", "fold"):
        for ps in ("exact", "p16"):
            out = emulate(flat, ids, lens, g, mode, ps, pooling=a.pooling)
            print(f"  emulated {mode:8s} l={ps:5s} vs fp64: {R.rel_l2(out, ref).max():.3e}   vs HF fp32: {R.rel_l2(out, hf).max():.3e}")
    if a.ablate:
        for keep in (("x",), ("w",), ("qkv",), ("p",), ("ctx",), ("ffn",), ("x", "w"), ("qkv", "p", "ctx"), ("x", "w", "qkv", "p", "ctx", "ffn")):
            out = emulate(flat, ids, lens, g, "current", "p16", keep)
            print(f"  fp32 kept at {'+'.join(keep):22s}: {R.rel_l2(out, ref).max():.3e}")


if __name__ == "__main__":
    main()
