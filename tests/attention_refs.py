"""fp64 reference of the attention kernel at any head size (12 heads of 64 for bge-base, 12 of 32 for bge-small), with the
same elementwise tolerance as kernel_refs.attention_ref -- each term next to the rounding it comes from -- written for a
head dim d: the scores are sums of d fp16 products and the softmax scale is 1 / sqrt(d).  At d = 64 it is
kernel_refs.attention_ref term for term."""
import numpy as np

from kernel_refs import SUB16, U16, U32, acc_ulps, check


def attention_ref(qkv16, lens, B, S, heads=12, head_dim=32, rows=None):
    """ctx [B*S, heads * head_dim] in fp64 (keys >= len masked, len clamped to [1, S] as the kernel does) and its tolerance.
    `rows`: for each item, the query rows (within the item, ascending) to compute; the result then holds those rows, item
    after item."""
    qkv = np.asarray(qkv16, np.float16).reshape(B, S, 3, heads, head_dim)
    scale = 1.0 / np.sqrt(head_dim)
    L = np.clip(np.asarray(lens, np.int64), 1, S)
    ctx_all, tol_all = [], []
    for b in range(B):  # one item at a time: [heads, S, S] fp64 score arrays
        n = int(L[b])
        x = qkv[b].astype(np.float64)
        qq = (x[:, 0] if rows is None else x[np.asarray(rows[b], np.int64), 0]).transpose(1, 0, 2)  # [heads, S, head_dim]
        kk, vv = (x[:n, j].transpose(1, 0, 2) for j in (1, 2))  # valid keys only: [heads, n, head_dim]
        s = qq @ kk.transpose(0, 2, 1)
        s_tol = acc_ulps(head_dim) * U32 * (np.abs(qq) @ np.abs(kk).transpose(0, 2, 1)) + 2.0 * U32 * np.abs(s)  # + the fma into ex2
        e = np.exp((s - s.max(-1, keepdims=True)) * scale)
        p = e / e.sum(-1, keepdims=True)
        ctx = p @ vv
        pv = p @ np.abs(vv)                                     # P . |V|
        spread = pv + np.abs(ctx)                               # bounds sum_j p_j |v_j - ctx|
        tol = (U16 * np.abs(ctx)                                # ctx rounded to fp16
               + U16 * pv                                       # P rounded to fp16 ...
               + SUB16 * p.max(-1, keepdims=True) * np.abs(vv).sum(-2, keepdims=True)  # ... absolutely, in the subnormal range
               + scale * s_tol.max(-1, keepdims=True) * spread  # score errors move P
               + (acc_ulps(n) + 16.0) * U32 * spread            # P.V and the row sum in fp32, ex2.approx, the rescales
               + SUB16)
        ctx_all.append(ctx.transpose(1, 0, 2).reshape(-1, heads * head_dim))
        tol_all.append(tol.transpose(1, 0, 2).reshape(-1, heads * head_dim))
    return np.concatenate(ctx_all), np.concatenate(tol_all)


def check_attention(what, ctx, qkv16, lens, B, S, heads=12, head_dim=32, rows=None):
    """`rows` as attention_ref's: ctx then holds those query rows only, item after item."""
    ref, tol = attention_ref(qkv16, lens, B, S, heads, head_dim, rows)
    got = np.asarray(ctx, np.float16).astype(np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output (padded query rows must stay finite too)"
    return check(what, got, ref, tol)
