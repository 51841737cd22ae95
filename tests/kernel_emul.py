"""Numpy emulations of what the CUDA kernels compute, rounding as they round: fp16 operands, fp32 accumulation and epilogues,
fp16 or hi + lo outputs.  They stand in for the kernels in the CPU tests that show a check discriminates: an emulation passes
the kernel_refs check, and a `mutant` standing for a plausible kernel bug fails it."""
import numpy as np

import kernel_refs as KR


def _pairwise(parts):
    """The kernels' pairwise combination of per-slice values: ((p0 + p1) + (p2 + p3)) + (p4 + p5) for six."""
    parts = list(parts)
    while len(parts) > 1:
        parts = [parts[i] + parts[i + 1] if i + 1 < len(parts) else parts[i] for i in range(0, len(parts), 2)]
    return parts[0]


def row_stats32(p, eps):
    """gemm_sm90.cu row_stats in fp32: (mean, rstd) of each row from its W / 128 (sum, M2) partials."""
    p = np.asarray(p, np.float32)
    s, m2 = p[..., 0], p[..., 1]
    P = s.shape[1]
    inv_n = np.float32(1.0 / (KR.SLICE * P))
    mean = _pairwise(s[:, i] for i in range(P)) * inv_n
    d = s * np.float32(1.0 / KR.SLICE) - mean[:, None]
    m = np.float32(KR.SLICE) * d * d + m2
    var = _pairwise(m[:, i] for i in range(P)) * inv_n
    return mean, (np.float32(1.0) / np.sqrt(var + np.float32(eps))).astype(np.float32)


def partials32(x, about_row_mean=False):
    """fp32 (sum, M2) partials per 128-column slice, M2 about the slice's own mean (or, as a mutant, the row's)."""
    sl = np.asarray(x, np.float32).reshape(x.shape[0], -1, KR.SLICE)
    mu = np.asarray(x, np.float32).mean(-1)[:, None, None] if about_row_mean else sl.mean(-1, keepdims=True)
    return np.stack([sl.sum(-1, dtype=np.float32), ((sl - mu) ** 2).sum(-1, dtype=np.float32)], -1)


def emulate_gemm(epi, a16, w16, bias, resid=None, ln_stats=None, ln_gamma=None, ln_beta=None, eps=1e-12, mutant=None,
                 resid_hilo=None, split=False):
    """The GEMM's rounding: fp16 operands, fp32 accumulation (k-blocks of 64 in reverse order), fp32 epilogue, fp16 or hi + lo
    out.  Epi 2 returns hi + lo as fp32 -- or, with `split`, (hi, lo, v) with v the fp32 value the row statistics are taken
    of; its residual is fp32 `resid` (split here) or the fp16 pair `resid_hilo`."""
    from scipy.special import erf

    K = a16.shape[1]
    a32, w32 = a16.astype(np.float32), w16.astype(np.float32)
    blocks = list(range(K // 64))[::-1]
    if mutant == "drop_kblock":
        blocks = blocks[1:]
    acc = np.zeros((a16.shape[0], w16.shape[0]), np.float32)
    for kb in blocks:
        acc += a32[:, kb * 64:(kb + 1) * 64] @ w32[:, kb * 64:(kb + 1) * 64].T
    bias = np.asarray(bias, np.float32)
    if mutant == "bias_shift":
        bias = np.roll(bias, 1)
    if epi != 2:
        v = acc + bias
        if ln_stats is not None:
            _, rstd = row_stats32(ln_stats, eps)
            v = rstd[:, None] * acc + bias
        gelu = {1: "erf", 3: "quick"}.get(epi)
        if mutant == "gelu_swap":
            gelu = {"erf": "quick", "quick": "erf"}[gelu]
        if gelu == "erf":
            v = (v * np.float32(0.5) * (np.float32(1.0) + erf(v / np.float32(np.sqrt(2.0))))).astype(np.float32)
        elif gelu == "quick":
            v = (v / (np.float32(1.0) + np.exp(np.float32(-1.702) * v))).astype(np.float32)
        out = v.astype(np.float16)
    else:
        hi, lo = resid_hilo if resid_hilo is not None else KR.split_hilo(resid)
        r = hi.astype(np.float32) + lo.astype(np.float32)
        if ln_stats is not None:
            mean, rstd = row_stats32(ln_stats, eps)
            r = ((r - mean[:, None]) * rstd[:, None]) * np.asarray(ln_gamma, np.float32) + np.asarray(ln_beta, np.float32)
        v = acc + bias + r
        h2, l2 = KR.split_hilo(v)
        if split:
            return h2, l2, v
        out = h2.astype(np.float32) + (0 if mutant == "lo_dropped" else l2.astype(np.float32))
    if mutant == "swap_halves":  # the two consumer warpgroups' 64-row halves of every 128-row tile exchanged
        out = out.reshape(-1, 2, 64, out.shape[1])[:, ::-1].reshape(out.shape)
    if mutant == "permute_fragments":  # 8-column fragments j and j + 1 exchanged inside every 256-column tile
        out = out.reshape(out.shape[0], -1, 16, 2, 8)[:, :, :, ::-1].reshape(out.shape)
    return out


def emulate_attention(qkv16, lens, B, S, mutant=None, head_dim=64, heads=12, causal=False):
    """attention_sm90.cu's rounding: fp32 scores, online softmax over 64-key sub-blocks with exp2, P rounded to fp16, fp32
    P.V, ctx = fp16(O / l).  `heads` heads of head_dim.  `causal`: a query row skips the sub-blocks that start after it and
    masks the keys after it in the sub-block it sits in (the diagonal one)."""
    c = np.float32(1.4426950408889634 / np.sqrt(head_dim))
    H = heads * head_dim
    q = qkv16.reshape(B, S, 3, heads, head_dim).astype(np.float32)
    ctx = np.zeros((B, S, heads, head_dim), np.float16)
    for b in range(B):
        n = int(min(max(lens[b], 1), S)) + {"mask_plus": 1, "mask_minus": -1}.get(mutant, 0)
        qq, kk, vv = (q[b, :, j].transpose(1, 0, 2) for j in range(3))
        o = np.zeros((heads, S, head_dim), np.float32)
        m = np.full((heads, S, 1), -np.inf, np.float32)
        l = np.zeros((heads, S, 1), np.float32)
        for k0 in range(0, n, 64):
            r = slice(k0, S) if causal else slice(0, S)  # the query rows that read this sub-block
            s = qq[:, r] @ kk[:, k0:k0 + 64].transpose(0, 2, 1)
            s[:, :, max(n - k0, 0):] = -np.inf
            if causal:
                nr, nk = min(64, s.shape[1]), s.shape[2]
                s[:, :nr][:, np.arange(nk)[None, :] > np.arange(nr)[:, None]] = -np.inf
            m_new = np.maximum(m[:, r], s.max(-1, keepdims=True))
            alpha = np.exp2((m[:, r] - m_new) * c).astype(np.float32)
            if mutant == "no_rescale":
                alpha = np.where(np.isinf(m[:, r]), 0.0, 1.0).astype(np.float32)
            p = np.exp2(s * c - m_new * c).astype(np.float32)
            l[:, r] = l[:, r] * alpha + p.sum(-1, keepdims=True)
            o[:, r] = o[:, r] * alpha + p.astype(np.float16).astype(np.float32) @ vv[:, k0:k0 + 64]
            m[:, r] = m_new
        ctx[b] = (o / l).astype(np.float16).transpose(1, 0, 2)
    return ctx.reshape(B * S, H)


def ln32(x, g, b, eps):
    """The row kernels' two-pass fp32 LayerNorm."""
    x = np.asarray(x, np.float32)
    mu = x.mean(-1, keepdims=True, dtype=np.float32)
    d = x - mu
    rstd = np.float32(1.0) / np.sqrt((d * d).mean(-1, keepdims=True, dtype=np.float32) + np.float32(eps))
    return (d * rstd) * g + b


def l2_normalise32(z):
    z = np.asarray(z, np.float32)
    return z / np.maximum(np.linalg.norm(z, axis=-1, keepdims=True), np.float32(1e-12))


def fold_ln32(w, gamma=None, beta=None, bias=None):
    """The load-time fold in fp32 (fold_ln_kernel): (fp16(w o gamma - rowmean(w o gamma)), w beta + bias); without gamma
    (fp16(w), None)."""
    w = np.asarray(w, np.float32)
    if gamma is None:
        return w.astype(np.float16), None
    wg = w * np.asarray(gamma, np.float32)
    cv = (w @ np.asarray(beta, np.float32)).astype(np.float32)
    if bias is not None:
        cv = cv + np.asarray(bias, np.float32)
    return (wg - wg.mean(1, keepdims=True, dtype=np.float32)).astype(np.float16), cv
