"""fp64 references of what each CUDA kernel computes, and the one place the kernel-level tolerances are set.

A reference here takes the exact operands the kernel sees (fp16 bit patterns, the hi + lo residual, the (sum, M2) partials
it is handed) and computes the same operation in fp64.  Its tolerance is elementwise, a sum of bounds, each written next to
the rounding it comes from:

  * fp16 output rounding (round to nearest even): 2^-11 |x|, or 2^-25 absolute in the subnormal range;
  * fp32 accumulation of fp16 x fp16 products (exact in fp32) on the tensor core: ACC_ULPS(K) * 2^-24 * (|A| . |W|^T),
    elementwise -- a bound on the sum of absolute products, never a flat absolute term;
  * the residual stream y = hi + lo (two fp16): lo is itself rounded, 2^-22 relative, written 2^-21 for margin;
  * fp32 epilogue and row-kernel arithmetic: a counted number of 2^-24 roundings of the magnitudes that go in;
  * attention: P rounded to fp16 before P.V, 2^-11 (P . |V|); ctx rounded to fp16, 2^-11 |ctx|.

Every `check_*` goes through `check`, which prints the largest error and the margin (worst err / tol: < 1 passes)."""
import numpy as np

U16 = 2.0 ** -11   # fp16 unit roundoff, round to nearest
U32 = 2.0 ** -24   # fp32 unit roundoff
SUB16 = 2.0 ** -25  # half the fp16 subnormal spacing: the absolute rounding error below fp16's normal range
HILO = 2.0 ** -21  # y = hi + lo against the fp32 value it was split from
H = 768
SLICE = 128        # row statistics travel as one (sum, M2) partial per 128 columns


def acc_ulps(K):
    """fp32 accumulation over K fp16 products, in units of 2^-24 * sum_k |a_k w_k|.  The tensor core adds the products in
    small groups, aligning to the largest term and truncating, so every group can lose up to one fp32 ulp of the running
    sum, with a common sign.  For the zero-mean operands of these layers the running sum grows like sqrt(k) * |a||w|, so
    the K/4 group roundings stay below ~0.5 sqrt(K) * 2^-24 * sum |a w|; 2 sqrt(K) + 8 leaves a factor of four."""
    return 2.0 * np.sqrt(K) + 8.0


def check(what, got, ref, tol):
    """|got - ref| <= tol everywhere (NaN fails).  Prints the largest error and the margin; returns the margin."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    tol = np.broadcast_to(np.asarray(tol, np.float64), ref.shape)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = np.abs(got - ref)
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(err == 0, 0.0, err / tol)
    bad = ~(err <= tol)
    margin = float(np.nanmax(np.where(np.isnan(ratio), np.inf, ratio))) if ratio.size else 0.0
    print(f"{what}: max |err| {float(np.nanmax(err)) if err.size else 0.0:.3e}, worst err/tol {margin:.3f}")
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} outside tolerance, first at {np.argwhere(bad)[:4].tolist()}, worst err/tol {margin:.3g}"
    return margin


def fp16_round_tol(x):
    """fp16 round-to-nearest of a value of magnitude |x|."""
    return U16 * np.abs(x) + SUB16


def ulp16(x):
    """Spacing of fp16 at |x| (2^-24 in the subnormal range)."""
    a = np.abs(np.asarray(x, np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def split_hilo(x32):
    """The host / kernel split of an fp32 value into the residual stream: hi = fp16(x), lo = fp16(x - hi)."""
    x32 = np.asarray(x32, np.float32)
    hi = x32.astype(np.float16)
    lo = (x32 - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def hilo64(hi, lo):
    return hi.astype(np.float64) + lo.astype(np.float64)


# ------------------------------------------------------------------------------------------------ row statistics

def partials(y):
    """(sum, M2 about the slice's own mean) per 128-column slice, fp64: [rows, W/128, 2]."""
    y = np.asarray(y, np.float64)
    sl = y.reshape(y.shape[0], -1, SLICE)
    s = sl.sum(-1)
    m2 = ((sl - sl.mean(-1, keepdims=True)) ** 2).sum(-1)
    return np.stack([s, m2], -1)


def partials_tol(y, ty, sum_ulps):
    """Tolerance of fp32 (sum, M2) partials of values y (fp64 reference) that the kernel holds with elementwise error <= ty,
    summed with `sum_ulps` sequential fp32 roundings per partial.  M2 is taken about the fp32 slice mean; to first order
    its error cancels (sum (y - mean) = 0), leaving 128 dmean^2."""
    y = np.asarray(y, np.float64)
    sl = y.reshape(y.shape[0], -1, SLICE)
    t = np.broadcast_to(np.asarray(ty, np.float64), y.shape).reshape(sl.shape)
    mu = sl.mean(-1, keepdims=True)
    d = np.abs(sl - mu)
    s_tol = t.sum(-1) + sum_ulps * U32 * np.abs(sl).sum(-1)
    dmu = s_tol / SLICE + U32 * np.abs(mu[..., 0])
    m2 = (d ** 2).sum(-1)
    m2_tol = 2.0 * (d * (t + 2.0 * U32 * (np.abs(sl) + np.abs(mu)))).sum(-1) + SLICE * dmu ** 2 + sum_ulps * U32 * m2
    return np.stack([s_tol, m2_tol], -1)


def check_partials(what, got, y, ty=0.0, sum_ulps=8):
    got = np.asarray(got, np.float64).reshape(-1, np.asarray(y).shape[1] // SLICE, 2)
    return check(what, got, partials(y), partials_tol(y, ty, sum_ulps))


def stats_from_partials(p, eps):
    """LayerNorm (mean, rstd) of each row from its partials, fp64 -- what the GEMM epilogue's row_stats computes -- and the
    error bounds of the kernel's fp32 combination: (mean, rstd, mean_tol, rstd_rel_tol), each [rows]."""
    p = np.asarray(p, np.float64)
    s, m2 = p[..., 0], p[..., 1]
    n = SLICE * s.shape[1]
    mean = s.sum(-1) / n
    d = s / SLICE - mean[:, None]
    var = (m2 + SLICE * d * d).sum(-1) / n
    rstd = 1.0 / np.sqrt(var + eps)
    mean_tol = 4.0 * U32 * np.abs(s).sum(-1) / n
    # d = s_i/128 - mean carries ~3 ulps of |mean|; 128 d^2 then moves by 256 |d| of that; plus the fp32 sums themselves
    var_tol = 8.0 * U32 * var + 6.0 * U32 * np.abs(mean) * np.abs(d).max(-1) * 2.0
    rstd_rel = 0.5 * var_tol / (var + eps) + 2.0 * U32  # + rsqrtf
    return mean, rstd, mean_tol, rstd_rel


# ------------------------------------------------------------------------------------------------ GEMM

def gelu_erf(x):
    from scipy.special import erf

    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def gelu_quick(x):
    return x / (1.0 + np.exp(-1.702 * x))


GELU_SLOPE = 1.13  # max |d gelu / dx| of both GELUs (erf: 1.129 at x = 1.5; quick: 1.10): how far an input error travels
GELU_ULPS = 8      # the kernels' GELUs: erf by Abramowitz-Stegun 7.1.26 (1.5e-7 absolute), rcp / ex2 .approx (2 ulp each)


def gemm_ref(epi, a16, w16, bias, resid=None, ln_stats=None, ln_gamma=None, ln_beta=None, eps=1e-12, resid_hilo=None):
    """What b200rt_debug_gemm returns, in fp64, and its elementwise tolerance: (ref, tol, v_tol), v_tol being the bound
    on the kernel's fp32 epilogue value before its output rounding (what the emitted row statistics are taken of).
    epi 2 takes the residual either as fp32 `resid`, split here as the debug entry splits it, or as the (hi, lo) fp16 pair
    `resid_hilo` the kernel read in place (a residual stream traced out of a forward: re-splitting hi + lo can move hi when
    lo sits exactly on half an ulp)."""
    a = np.asarray(a16, np.float16).astype(np.float64)
    w = np.asarray(w16, np.float16).astype(np.float64)
    K = a.shape[1]
    bias = np.asarray(bias, np.float32).astype(np.float64)
    acc = a @ w.T
    acc_tol = acc_ulps(K) * U32 * (np.abs(a) @ np.abs(w).T)
    if epi != 2:
        if ln_stats is not None:
            _, rstd, _, rstd_rel = stats_from_partials(ln_stats, eps)
            rstd, rstd_rel = rstd[:, None], rstd_rel[:, None]
        else:
            rstd, rstd_rel = 1.0, 0.0
        v = rstd * acc + bias
        v_tol = rstd * acc_tol + np.abs(rstd * acc) * rstd_rel + 2.0 * U32 * (np.abs(v) + np.abs(bias))
        if epi == 1:
            v, v_tol = gelu_erf(v), GELU_SLOPE * v_tol + GELU_ULPS * U32 * np.abs(v)
        elif epi == 3:
            v, v_tol = gelu_quick(v), GELU_SLOPE * v_tol + GELU_ULPS * U32 * np.abs(v)
        return v, v_tol + fp16_round_tol(np.abs(v) + v_tol), v_tol
    hi, lo = resid_hilo if resid_hilo is not None else split_hilo(resid)
    r = hilo64(np.asarray(hi, np.float16), np.asarray(lo, np.float16))  # the residual as the kernel holds it
    if ln_stats is not None:
        mean, rstd, mean_tol, rstd_rel = (x[:, None] for x in stats_from_partials(ln_stats, eps))
        g = np.asarray(ln_gamma, np.float32).astype(np.float64)
        b = np.asarray(ln_beta, np.float32).astype(np.float64)
        z = (r - mean) * rstd
        ln = z * g + b
        ln_tol = np.abs(g) * (rstd * (2.0 * U32 * (np.abs(r) + np.abs(mean)) + mean_tol) + np.abs(z) * (rstd_rel + 2.0 * U32)) + U32 * np.abs(ln)
    else:
        ln, ln_tol = r, 0.0
    v = acc + bias + ln
    v_tol = acc_tol + ln_tol + 3.0 * U32 * (np.abs(acc) + np.abs(bias) + np.abs(ln))
    return v, v_tol + HILO * (np.abs(v) + v_tol) + SUB16, v_tol


def check_gemm(what, out, epi, a16, w16, bias, **kw):
    ref, tol, _ = gemm_ref(epi, a16, w16, bias, **kw)
    return check(what, out, ref, tol)


def check_gemm_stats(what, stats_out, epi_args, **kw):
    """stats_out of the residual epilogue: (sum, M2) partials of the new fp32 rows, 16 pairs summed per thread, then
    reduced over the quad (2 shuffles): 20 roundings."""
    ref, _, v_tol = gemm_ref(2, *epi_args, **kw)
    return check_partials(what, stats_out, ref, v_tol, sum_ulps=20)


# ------------------------------------------------------------------------------------------------ attention

def attention_ref(qkv16, lens, B, S, rows=None):
    """ctx [B*S, 768] in fp64 (keys >= len masked, len clamped to [1, S] as the kernel does) and its tolerance.  `rows`: for
    each item, the query rows (within the item, ascending) to compute; the result then holds those rows, item after item."""
    qkv = np.asarray(qkv16, np.float16).reshape(B, S, 3, 12, 64)
    L = np.clip(np.asarray(lens, np.int64), 1, S)
    ctx_all, tol_all = [], []
    for b in range(B):  # one item at a time: [12, S, S] fp64 score arrays
        n = int(L[b])
        x = qkv[b].astype(np.float64)
        qq = (x[:, 0] if rows is None else x[np.asarray(rows[b], np.int64), 0]).transpose(1, 0, 2)  # [12, S, 64]
        kk, vv = (x[:n, j].transpose(1, 0, 2) for j in (1, 2))  # valid keys only: [12, n, 64]
        s = qq @ kk.transpose(0, 2, 1)
        s_tol = acc_ulps(64) * U32 * (np.abs(qq) @ np.abs(kk).transpose(0, 2, 1)) + 2.0 * U32 * np.abs(s)  # + the fma into ex2
        e = np.exp((s - s.max(-1, keepdims=True)) * 0.125)
        p = e / e.sum(-1, keepdims=True)
        ctx = p @ vv
        pv = p @ np.abs(vv)                                     # P . |V|
        spread = pv + np.abs(ctx)                               # bounds sum_j p_j |v_j - ctx|
        tol = (U16 * np.abs(ctx)                                # ctx rounded to fp16
               + U16 * pv                                       # P rounded to fp16 ...
               + SUB16 * p.max(-1, keepdims=True) * np.abs(vv).sum(-2, keepdims=True)  # ... absolutely, in the subnormal range
               + 0.125 * s_tol.max(-1, keepdims=True) * spread  # score errors move P
               + (acc_ulps(n) + 16.0) * U32 * spread            # P.V and the row sum in fp32, ex2.approx, the rescales
               + SUB16)
        ctx_all.append(ctx.transpose(1, 0, 2).reshape(-1, H))
        tol_all.append(tol.transpose(1, 0, 2).reshape(-1, H))
    return np.concatenate(ctx_all), np.concatenate(tol_all)


def check_attention(what, ctx, qkv16, lens, B, S, rows=None):
    """`rows` as attention_ref's: ctx then holds those query rows only, item after item."""
    ref, tol = attention_ref(qkv16, lens, B, S, rows)
    got = np.asarray(ctx, np.float16).astype(np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output (padded query rows must stay finite too)"
    return check(what, got, ref, tol)


# ------------------------------------------------------------------------------------------------ row kernels

LN_SUM_ULPS = 24  # a row sum in the row kernels: 6 float4 per lane (3 adds each, accumulated), then 5 butterfly levels


def layernorm_ref(x, g, b, eps):
    """fp64 LayerNorm of rows x and the bound on the fp32 two-pass LayerNorm of the same rows (the row kernels' ln_inplace):
    (y, y_tol, z) with z the normalised rows before gamma / beta."""
    x = np.asarray(x, np.float64)
    g = np.asarray(g, np.float32).astype(np.float64)
    b = np.asarray(b, np.float32).astype(np.float64)
    mu = x.mean(-1, keepdims=True)
    d = x - mu
    var = (d ** 2).mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + eps)
    z = d * rstd
    y = z * g + b
    mu_tol = LN_SUM_ULPS * U32 * np.abs(x).mean(-1, keepdims=True)
    d_tol = mu_tol + U32 * (np.abs(x) + np.abs(mu))
    var_tol = 2.0 * (np.abs(d) * d_tol).mean(-1, keepdims=True) + LN_SUM_ULPS * U32 * var
    rstd_rel = 0.5 * var_tol / (var + eps) + 2.0 * U32
    y_tol = np.abs(g) * (rstd * d_tol + np.abs(z) * (rstd_rel + 2.0 * U32)) + 2.0 * U32 * np.abs(y)
    return y, y_tol, z


def embed_exact(ids, word, pos, type0, S):
    """embed_kernel, bit for bit: x = (word[id] + type0) + pos[t % S] in fp32 (HF's order), hi = fp16_rn(x),
    lo = fp16_rn(x - hi).  Returns (hi, lo, x)."""
    ids = np.asarray(ids).reshape(-1)
    t = np.arange(ids.size)
    x = (np.asarray(word, np.float32)[ids] + np.asarray(type0, np.float32)[None, :]) + np.asarray(pos, np.float32)[t % S]
    hi, lo = split_hilo(x)
    return hi, lo, x


def check_bits(what, got, want):
    """Bitwise equality of fp16 arrays (so -0 / +0 and the infinities count)."""
    g = np.asarray(got, np.float16).view(np.uint16)
    w = np.asarray(want, np.float16).view(np.uint16)
    bad = g != w
    print(f"{what}: {int(bad.sum())} of {bad.size} fp16 values differ bitwise")
    assert not bad.any(), f"{what}: first differing at {np.argwhere(bad)[:4].tolist()}: got {g[bad][:4]}, want {w[bad][:4]}"


def check_embed(what, hi, lo, stats, ids, word, pos, type0, S, rows=None):
    """hi and lo bit for bit over every row; the partials over `rows` (stats then holds those rows), by default all."""
    hi_r, lo_r, x = embed_exact(ids, word, pos, type0, S)
    check_bits(f"{what} hi", hi, hi_r)
    check_bits(f"{what} lo", lo, lo_r)
    if rows is not None:
        x = x[rows]
    fin = np.isfinite(x).all(-1)  # rows that overflow fp32 have no meaningful statistics
    return check_partials(f"{what} partials", np.asarray(stats)[fin], x[fin].astype(np.float64))


def hi_is_nearest(what, hi, lo):
    """hi is an fp16 nearest to hi + lo: |lo| <= half an ulp of hi (lo is itself rounded, so it can land exactly on the half
    ulp with hi odd; fp16(hi + lo) would then round to the even neighbour)."""
    h = np.asarray(hi, np.float16)
    l = np.abs(np.asarray(lo, np.float16).astype(np.float64))
    bad = ~(l <= 0.5 * ulp16(h.astype(np.float64)))
    exact = np.asarray((h.astype(np.float64) + np.asarray(lo, np.float16).astype(np.float64)).astype(np.float16) == h)
    print(f"{what}: hi == fp16(hi + lo) for {exact.mean() * 100:.3f} % of values, |lo| <= half an ulp of hi everywhere: {not bad.any()}")
    assert not bad.any(), f"{what}: |lo| exceeds half an ulp of hi at {np.argwhere(bad)[:4].tolist()}"


def vit_embed_ref(patch16, cls, pos, gamma, beta, T, eps):
    """pre_layrnorm((class token | fp16 patch row) + position), fp64: (y, y_tol) for the fp32 value the kernel splits."""
    rows = np.asarray(patch16).shape[0]
    tk = np.arange(rows) % T
    src = np.where((tk == 0)[:, None], np.asarray(cls, np.float32).astype(np.float64)[None, :], np.asarray(patch16, np.float16).astype(np.float64))
    x = src + np.asarray(pos, np.float32).astype(np.float64)[tk]
    y, y_tol, _ = layernorm_ref(x, gamma, beta, eps)
    y_tol = y_tol + np.abs(np.asarray(gamma, np.float64)) * U32 * np.abs(x) / np.sqrt(x.var(-1, keepdims=True) + eps)  # the fp32 add
    return y, y_tol


def check_vit_embed(what, hi, lo, stats, patch16, cls, pos, gamma, beta, T, eps):
    y, y_tol = vit_embed_ref(patch16, cls, pos, gamma, beta, T, eps)
    m = check(f"{what} hi+lo", hilo64(hi, lo), y, y_tol + HILO * np.abs(y) + SUB16)
    hi_is_nearest(what, hi, lo)
    check_partials(f"{what} partials", stats, y, y_tol, sum_ulps=8)
    return m


def _normalised(v, v_tol, norm_ulps):
    """L2-normalise rows v (fp64) whose kernel values carry error <= v_tol; the fp32 norm adds `norm_ulps` roundings."""
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    out = v / np.maximum(n, 1e-12)
    dn = np.linalg.norm(v_tol, axis=-1, keepdims=True) + norm_ulps * U32 * n
    tol = (v_tol + np.abs(out) * dn) / np.maximum(n, 1e-12) + 2.0 * U32 * np.abs(out)
    return out, tol


def pool_normalize_ref(hi, lo, gamma, beta, S, eps):
    x = hilo64(hi, lo)[::S]
    y, y_tol, _ = layernorm_ref(x, gamma, beta, eps)
    return _normalised(y, y_tol, LN_SUM_ULPS)


def check_pool_normalize(what, out, hi, lo, gamma, beta, S, eps):
    ref, tol = pool_normalize_ref(hi, lo, gamma, beta, S, eps)
    return check(what, out, ref, tol)


def vit_pool_ref(hi, lo, gamma, beta, proj, T, eps):
    x = hilo64(hi, lo)[::T]
    z, z_tol, _ = layernorm_ref(x, gamma, beta, eps)
    w = np.asarray(proj, np.float32).astype(np.float64)
    y = z @ w.T
    # 24 fma per lane + 5 butterfly levels per output, the LayerNorm's error carried through |W|
    y_tol = z_tol @ np.abs(w).T + 30.0 * U32 * (np.abs(z) @ np.abs(w).T)
    return _normalised(y, y_tol, 8 + LN_SUM_ULPS)


def check_vit_pool(what, out, hi, lo, gamma, beta, proj, T, eps):
    ref, tol = vit_pool_ref(hi, lo, gamma, beta, proj, T, eps)
    return check(what, out, ref, tol)


def fold_ln_ref(w, gamma, beta, bias):
    """Load-time fold: (w o gamma - rowmean(w o gamma), w beta + bias) in fp64, and cvec's tolerance (one lane: K/64 steps of
    two fma, then 5 butterfly levels and the bias add)."""
    w = np.asarray(w, np.float32).astype(np.float64)
    g = np.asarray(gamma, np.float32).astype(np.float64)
    be = np.asarray(beta, np.float32).astype(np.float64)
    bs = np.zeros(w.shape[0]) if bias is None else np.asarray(bias, np.float32).astype(np.float64)
    wg = w * g
    wf = wg - wg.mean(1, keepdims=True)
    c = w @ be + bs
    c_tol = (2 * w.shape[1] / 64 + 7) * U32 * (np.abs(w) @ np.abs(be) + np.abs(bs))
    return wf, c, c_tol


def check_fold_ln(what, w_out, cvec, w, gamma, beta, bias):
    """w_out within one fp16 ulp of the fp64 fold -- half an ulp of rounding plus the fp32 row mean, whose bound exceeds the
    other half only next to zero, where it is used instead -- and cvec within its fp32 bound."""
    wf, c, c_tol = fold_ln_ref(w, gamma, beta, bias)
    wg = np.abs(np.asarray(w, np.float64) * np.asarray(gamma, np.float64))
    K = wg.shape[1]
    mean_tol = (2 * K / 64 + 6) * U32 * wg.sum(1, keepdims=True) / K
    tol = np.maximum(ulp16(wf), 0.5 * ulp16(wf) + mean_tol + U32 * wg)
    m = check(f"{what} w_out", np.asarray(w_out, np.float16), wf, tol)
    check(f"{what} cvec", cvec, c, c_tol)
    return m
