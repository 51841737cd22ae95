"""Mean pooling (sentence-transformers ``Pooling(mean)`` + ``Normalize``), the way the tests see it:

  * the model-level oracle: the encoder of ``oracle/bge_ref.py`` followed by the masked mean of the last hidden states over
    each item's valid tokens ([CLS] and [SEP] included) and L2 normalisation -- in numpy fp64 (`forward_np_mean`) and in HF
    torch fp32 with sentence-transformers' own arithmetic (`forward_hf_mean`);
  * the fp64 reference of ``mean_pool_normalize_kernel`` and its tolerance (`mean_pool_normalize_ref`), built from the terms of
    ``kernel_refs``: the per-row LayerNorm bound of `layernorm_ref`, counted fp32 roundings of the row sum and of the warp
    combine, and `_normalised`;
  * a numpy emulation of the kernel, rounding as it rounds, with mutants standing for plausible kernel bugs
    (`emulate_mean_pool`)."""
import math

import numpy as np

import kernel_refs as KR
import kernel_emul as KE
from oracle import bge_ref as R

WARPS = 8           # mean_pool_normalize_kernel: one block of 8 warps per item, warp w sums rows w, w + 8, ...
COMBINE_ULPS = 7    # the 8 warp sums added in warp order
DIV_ULPS = 1        # sum / len
NORM_ULPS = 16      # sum of squares: <= 3 fma per thread, 5 butterfly levels, 7 adds over the warps


# ------------------------------------------------------------------------------------------------ model-level oracle

def _mean_normalise(h, lens):
    """Masked mean over the first lens[i] rows of h [B, S, H] (fp64), then L2 normalise (F.normalize eps 1e-12)."""
    B, S, _ = h.shape
    mask = (np.arange(S)[None, :] < np.asarray(lens)[:, None]).astype(np.float64)
    m = (h * mask[..., None]).sum(1) / np.maximum(mask.sum(1), 1e-9)[:, None]
    return (m / np.maximum(np.linalg.norm(m, axis=-1, keepdims=True), 1e-12)).astype(np.float32)


def forward_np_mean(flat, ids, lens=None, g=R.BGE_BASE, dtype=np.float64):
    """``bge_ref.forward_np``'s encoder (computed in `dtype`), mean-pooled over the valid tokens and L2-normalised.  The
    oracle hands its last hidden state out as float32; the mean and the norm are then taken in fp64 (the fp32 rounding of the
    hidden state is ~6e-8 relative, far below every bar this is used with)."""
    ids = np.asarray(ids)
    B, S = ids.shape
    lens = np.full(B, S, np.int32) if lens is None else np.asarray(lens)
    _, hidden = R.forward_np(flat, ids, lens, g, dtype=dtype, return_hidden=True)
    return _mean_normalise(hidden[-1].astype(np.float64), lens)


def forward_hf_mean(model, ids, lens=None):
    """HF ``BertModel`` (fp32 CPU) + sentence-transformers' Pooling(mean) + Normalize in torch:
    ``(h * mask).sum(1) / mask.sum(1).clamp(min=1e-9)``, then ``F.normalize``."""
    import torch

    ids_t = torch.from_numpy(np.ascontiguousarray(ids)).long()
    B, S = ids_t.shape
    if lens is None:
        mask = torch.ones(B, S, dtype=torch.long)
    else:
        mask = (torch.arange(S)[None, :] < torch.from_numpy(np.asarray(lens))[:, None]).long()
    with torch.no_grad():
        h = model(input_ids=ids_t, attention_mask=mask, token_type_ids=torch.zeros_like(ids_t)).last_hidden_state
        m = mask.unsqueeze(-1).expand(h.size()).float()
        emb = (h * m).sum(1) / m.sum(1).clamp(min=1e-9)
        emb = torch.nn.functional.normalize(emb, p=2, dim=1)
    return emb.numpy().astype(np.float32)


# ------------------------------------------------------------------------------------------------ kernel reference

def row_sum_ulps(L):
    """fp32 roundings of one warp's running row sum: it adds ceil(L / 8) rows."""
    return math.ceil(L / WARPS)


def mean_pool_normalize_ref(hi, lo, gamma, beta, lens, S, eps):
    """What b200rt_debug_mean_pool_normalize returns, in fp64, and its elementwise tolerance: (ref, tol), [n_items, W].
    Each item's rows r < L (L = lens[i] clamped to [1, S], as the kernel clamps) are LayerNorm'd with `layernorm_ref`'s bound,
    averaged -- the row sum and the warp combine each adding counted fp32 roundings of sum |y|, the division one more of the
    mean -- and L2-normalised by `_normalised`.  Rows past L do not enter."""
    W = np.asarray(hi).shape[1]
    x = KR.hilo64(np.asarray(hi, np.float16), np.asarray(lo, np.float16)).reshape(-1, S, W)
    L = np.clip(np.asarray(lens, np.int64), 1, S)
    means, tols = np.empty((len(L), W)), np.empty((len(L), W))
    for i, n in enumerate(L):
        n = int(n)
        y, y_tol, _ = KR.layernorm_ref(x[i, :n], gamma, beta, eps)
        m = y.mean(0)
        means[i] = m
        tols[i] = y_tol.mean(0) + (row_sum_ulps(n) + COMBINE_ULPS) * KR.U32 * np.abs(y).mean(0) + DIV_ULPS * KR.U32 * np.abs(m)
    return KR._normalised(means, tols, NORM_ULPS)


def check_mean_pool_normalize(what, out, hi, lo, gamma, beta, lens, S, eps):
    ref, tol = mean_pool_normalize_ref(hi, lo, gamma, beta, lens, S, eps)
    return KR.check(what, out, ref, tol)


# ------------------------------------------------------------------------------------------------ kernel emulation

MUTANTS = ("unmasked_mean", "padding_row", "drop_cls", "average_then_ln", "stop_short")
# Dividing the masked sum by S instead of len scales each item by len / S, which Normalize removes: the output is the same
# to within rounding, so that mutant is equivalent, not a bug the output could show (the CPU test keeps it as such).
EQUIVALENT_MUTANTS = ("divide_by_S",)


def emulate_mean_pool(hi, lo, gamma, beta, lens, S, eps, mutant=None):
    """mean_pool_normalize_kernel's rounding: y = hi + lo in fp32, the fp32 two-pass LayerNorm of each valid row, warp w's
    fp32 sum of rows w, w + 8, ..., the 8 warp sums added in order, / len, fp32 L2 normalise.  Mutants: divide by S instead
    of len (equivalent, see EQUIVALENT_MUTANTS), the unmasked mean over all S rows, include the first padding row, drop the
    [CLS] row, average the raw rows first and LayerNorm the mean, stop one row short.  (Using the wrong LayerNorm is
    emulated by passing that LayerNorm's parameters.)"""
    W = np.asarray(hi).shape[1]
    x = (np.asarray(hi, np.float16).astype(np.float32) + np.asarray(lo, np.float16).astype(np.float32)).reshape(-1, S, W)
    g, b = np.asarray(gamma, np.float32), np.asarray(beta, np.float32)
    out = np.empty((x.shape[0], W), np.float32)
    for i, n in enumerate(np.clip(np.asarray(lens, np.int64), 1, S)):
        n = int(n)
        lo_r, hi_r, denom = 0, n, n
        if mutant == "divide_by_S":
            denom = S
        elif mutant == "unmasked_mean":
            hi_r, denom = S, S
        elif mutant == "padding_row":
            hi_r = min(n + 1, S)
        elif mutant == "drop_cls":
            lo_r = 1
        elif mutant == "stop_short":
            hi_r = n - 1
        rows = x[i, lo_r:hi_r]
        if mutant == "average_then_ln":
            m = KE.ln32(rows.mean(0, dtype=np.float32)[None], g, b, eps)[0]
        else:
            y = KE.ln32(rows, g, b, eps) if len(rows) else np.zeros((0, W), np.float32)
            acc = np.zeros((WARPS, W), np.float32)
            for k0 in range(0, len(y), WARPS):
                blk = y[k0:k0 + WARPS]
                acc[:len(blk)] += blk
            s = acc[0].copy()
            for w in range(1, WARPS):
                s = s + acc[w]
            m = s / np.float32(denom)
        out[i] = KE.l2_normalise32(m[None])[0]
    return out
