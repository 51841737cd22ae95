"""Kernel conformance: every GEMM epilogue, launch-shape invariance, the split-SM runtime, the row kernels and attention cases
with an exact answer, each against an fp64 reference (tests/kernel_refs.py) at the tolerance its rounding implies.

The GPU tests carry `@gpu`.  The tests without it run on the CPU and show that each check discriminates: a numpy emulation
of the kernel's rounding passes it, and each mutant standing for a plausible kernel bug -- a dropped k-block, swapped tile
halves, permuted fragments, a shifted bias, the wrong GELU, a dropped lo, a partial about the wrong mean, an off-by-one key
mask or position, a missing rescale, the wrong pooled row -- fails it."""
import numpy as np
import pytest

import kernel_emul as KE
import kernel_refs as KR

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _ln_inputs(rng, M, W, mean=0.3, std=1.7):
    y = (rng.standard_normal((M, W)) * std + mean).astype(np.float32)
    y += np.repeat(rng.standard_normal(W // 64) * 0.5, 64)[None, :].astype(np.float32)  # slices with their own means
    g = (1.0 + 0.3 * rng.standard_normal(W)).astype(np.float32)
    b = (0.2 * rng.standard_normal(W)).astype(np.float32)
    return y, g, b


def _gemm_case(epi, M, N, K, seed, ln=None):
    """Operands of one debug_gemm call: epi 0/1/3 fold a LayerNorm of the A rows (W centred), epi 2 re-applies one to the
    residual -- when that row is 768 wide, the only LayerNorm width the kernel takes; returns (args, kwargs) for both
    debug_gemm and kernel_refs.gemm_ref."""
    if ln is None:
        ln = (N if epi == 2 else K) == KR.H
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    kw = dict(eps=1e-12)
    if epi == 2:
        a = rng.standard_normal((M, K)).astype(np.float16)
        resid, g, b = _ln_inputs(rng, M, N, mean=-0.5, std=2.0)
        kw["resid"] = resid
        if ln:
            kw.update(ln_stats=KR.partials(KR.hilo64(*KR.split_hilo(resid))).astype(np.float32), ln_gamma=g, ln_beta=b)
    else:
        y, _, _ = _ln_inputs(rng, M, K)
        a = y.astype(np.float16)
        if ln:
            w = (w.astype(np.float32) - w.astype(np.float32).mean(1, keepdims=True)).astype(np.float16)
            kw["ln_stats"] = KR.partials(y).astype(np.float32)
    return (a, w, bias), kw


# ================================================================================================ launch-shape invariance

@gpu
@pytest.mark.parametrize("epi", [0, 1, 2, 3])
def test_gemm_launch_shape_invariance(rt, epi):
    """297 / 291 tiles (33 x 9; epi 2, whose LayerNorm'd rows are 768 wide, 97 x 3), the last row tile 4 / 12 rows deep, on
    1, 2, 7, 66, 131 CTAs: outputs (and epi 2's row statistics) bitwise equal to the launch on every SM.  On one CTA the
    4-stage ring wraps over 3400 times."""
    M, N, K = (12300, 768, 768) if epi == 2 else (4100, 2304, 768)
    args, kw = _gemm_case(epi, M, N, K, seed=10 + epi)
    want = epi == 2
    base = rt.debug_gemm(epi, *args, want_stats=want, **kw)
    KR.check_gemm(f"epi {epi} sms 0", base[0], epi, *args, **kw)
    if want:
        KR.check_gemm_stats(f"epi {epi} stats_out", base[2], args, **kw)
    for sms in (1, 2, 7, 66, 131):
        got = rt.debug_gemm(epi, *args, want_stats=want, sms=sms, **kw)
        same = np.array_equal(got[0].view(np.uint32 if epi == 2 else np.uint16), base[0].view(np.uint32 if epi == 2 else np.uint16))
        same_st = not want or np.array_equal(got[2].view(np.uint32), base[2].view(np.uint32))
        print(f"epi {epi}: sms {sms} bitwise equal to sms 0: out {same}, stats {same_st}")
        assert same and same_st, sms


@gpu
def test_attention_launch_shape_invariance(rt):
    """B = 4 (48 units): the query-tile split starts above 48 SMs.  1 / 7 / 47 / 48 CTAs walk (item, head) units whose K/V
    tile counts differ (the kv_par parity bookkeeping), 49 / 132 walk query-tile units; every output is bitwise the same."""
    B, S, lens = 4, 512, [512, 77, 300, 129]
    rng = np.random.default_rng(4)
    qkv = (rng.standard_normal((B * S, 2304)) * 2.0).astype(np.float16)
    base, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S)
    KR.check_attention("attention sms 0", base, qkv, lens, B, S)
    for sms in (1, 7, 47, 48, 49, 132):
        got, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S, sms=sms)
        same = np.array_equal(got.view(np.uint16), base.view(np.uint16))
        print(f"attention: sms {sms} ({'split by query tile' if B * 12 < sms else 'one unit per head'}) bitwise equal to sms 0: {same}")
        assert same, sms
    with pytest.raises(rt.B200RTError) as e:
        rt.debug_attention(qkv, np.array(lens, np.int32), B, S, sms=10_000)
    assert e.value.code == rt.E_INVALID
    with pytest.raises(rt.B200RTError) as e:
        rt.debug_gemm(0, qkv[:128, :64], qkv[:256, :64], np.zeros(256, np.float32), sms=-1)
    assert e.value.code == rt.E_INVALID


@gpu
@pytest.mark.parametrize("k", [20, 66])
def test_split_sm_runtime_matches_whole_gpu(rt, k):
    """B200RT_INIT_SPLIT_SMS(k): two replicas on one GPU, GEMMs on 132 - k CTAs, attention on k.  A ragged text batch spread
    over both replicas and a ViT batch give the whole-GPU runtime's bits.  The module's runtime is shut down for the
    duration and restarted afterwards."""
    from oracle import bge_ref as R
    from oracle import clip_ref as C

    tg = R.BertGeometry(layers=2)
    tblob = R.pack_blob(R.make_weights(tg, 3, "trained"), tg)
    vg = C.VitGeometry(layers=2)
    vblob = C.pack_blob(C.make_weights(vg, 1, "trained"), vg)
    ids1, lens1 = R.synth_ragged(40, 192, seed=11, min_len=129)  # one 192-token bucket: 40 items, both replicas
    ids2, lens2 = R.synth_ragged(20, 512, seed=12, min_len=1)    # every bucket
    px = C.synth_pixels(24, vg, 3)

    def run(flags):
        rt.shutdown()
        rt.init(devices=[0], flags=flags)
        text = rt.EmbedModel(R.geometry_dict(tg), tblob)
        vit = rt.ImageEmbedModel(C.geometry_dict(vg), vblob)
        out = (text.embed(ids1, lens1), text.embed(ids2, lens2), vit.embed(px))
        return out, rt.num_gpus(), rt.stats()["peer_bytes"]

    try:
        whole, n_whole, _ = run(0)
        split, n_split, peer = run(rt.SPLIT_SMS(k))
    finally:
        rt.shutdown()
        rt.init(devices=[0])
    assert n_whole == 1 and n_split == 2
    assert peer > 0, "the second replica took no items"
    for name, a, b in zip(("text bucket 192", "text ragged", "vit"), whole, split):
        same = np.array_equal(a.view(np.uint32), b.view(np.uint32))
        print(f"split SMs k={k}: {name} ({a.shape[0]} items) bitwise equal to the whole-GPU runtime: {same}")
        assert same, name


# ================================================================================================ epilogue edges

@gpu
@pytest.mark.parametrize("epi", [1, 3])
def test_gelu_epilogue_tails(rt, epi):
    """Pre-activations swept over [-30, 30] through the bias: the negative tail is +-0 and never NaN, the positive tail is the
    pre-activation itself, the middle is within tolerance of the fp64 GELU."""
    M, N, K = 64, 4096, 64
    rng = np.random.default_rng(epi)
    a = rng.standard_normal((M, K)).astype(np.float16)
    w = (rng.standard_normal((N, K)) * 1e-3).astype(np.float16)
    bias = np.linspace(-30.0, 30.0, N).astype(np.float32)
    out, _ = rt.debug_gemm(epi, a, w, bias)
    KR.check_gemm(f"epi {epi} sweep", out, epi, a, w, bias)
    pre = a.astype(np.float64) @ w.astype(np.float64).T + bias
    o = out.astype(np.float64)
    assert not np.isnan(o).any()
    neg, pos = pre < -20.0, pre > 20.0
    assert (o[neg] == 0.0).all(), o[neg][o[neg] != 0][:4]
    assert (np.abs(o[pos] - pre[pos]) <= KR.ulp16(pre[pos])).all()
    print(f"epi {epi}: {int(neg.sum())} values below -20 all +-0, {int(pos.sum())} above 20 within an fp16 ulp of x")


@gpu
def test_residual_epilogue_without_layernorm_emits_statistics(rt):
    """CLIP's pre-LN residual: y' = acc + bias + y with stats_in = NULL, stats_out set (they feed the next LayerNorm fold),
    including rows with mean 150, std 1 -- the partials about each slice's own mean stay exact there."""
    M, N, K = 300, 768, 768
    rng = np.random.default_rng(21)
    a = rng.standard_normal((M, K)).astype(np.float16)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = (0.1 * rng.standard_normal(N)).astype(np.float32)
    resid = (rng.standard_normal((M, N)) * 2.0).astype(np.float32)
    resid[::3] = (150.0 + rng.standard_normal((len(resid[::3]), N))).astype(np.float32)
    out, _, st = rt.debug_gemm(2, a, w, bias, resid, want_stats=True)
    KR.check_gemm("residual, no LayerNorm", out, 2, a, w, bias, resid=resid)
    KR.check_gemm_stats("residual, no LayerNorm: stats_out", st, (a, w, bias), resid=resid)
    KR.check_gemm_stats("  rows with mean 150", st[::3], (a[::3], w, bias), resid=resid[::3])


# ================================================================================================ row kernels

def _embed_tables(rng, vocab, S):
    """Word / position / type tables whose sums hit the fp16 edges: the first 16 columns carry -0 in pos and type0, so word
    row 1 gives x = -0, row 2 fp16 subnormals, row 3 values that round to +-inf (and the largest finite fp16)."""
    word = (rng.standard_normal((vocab, KR.H)) + np.repeat(rng.standard_normal(6) * 3.0, 128)[None, :]).astype(np.float32)
    pos = rng.standard_normal((S, KR.H)).astype(np.float32)
    type0 = (0.3 * rng.standard_normal(KR.H)).astype(np.float32)
    pos[:, :16] = -0.0
    type0[:16] = -0.0
    word[1, :16] = -0.0
    word[2, :16] = (rng.standard_normal(16) * 2e-6).astype(np.float32)            # fp16 subnormals (< 6.1e-5)
    word[2, 0] = 2.0 ** -25                                                       # exactly half the smallest subnormal
    word[3, :16] = [70000, -70000, 65520, -65520, 65519, 65504, 1e5, -1e5, 65536, 2.0 ** -24, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11,
                    -(1 + 2.0 ** -11), 3e-8, -3e-8, 0.0]
    return word, pos, type0


@gpu
def test_embed_bit_exact_and_partials(rt):
    vocab, S, n_items = 64, 100, 3
    rng = np.random.default_rng(5)
    word, pos, type0 = _embed_tables(rng, vocab, S)
    ids = rng.integers(0, vocab, size=n_items * S).astype(np.int32)
    ids[:8] = [1, 2, 3, 1, 2, 3, 0, vocab - 1]
    hi, lo, st = rt.debug_embed(ids, word, pos, type0, S)
    KR.check_embed("embed", hi, lo, st, ids, word, pos, type0, S)


@gpu
def test_fold_ln_without_gamma_is_fp16_conversion(rt):
    rng = np.random.default_rng(6)
    w = rng.standard_normal((37, 192)).astype(np.float32)
    w[0, :16] = [70000, -70000, 65520, -65520, 65519, 65504, 1e30, -0.0, 0.0, 2.0 ** -25, 3 * 2.0 ** -26, 1e-7, -1e-7,
                 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 6.1e-5]
    w_out, cvec = rt.debug_fold_ln(w)
    assert cvec is None
    KR.check_bits("fold_ln(gamma=NULL)", w_out, w.astype(np.float16))


@gpu
def test_fold_ln_with_gamma(rt):
    rng = np.random.default_rng(7)
    N, K = 300, 768
    w = (rng.standard_normal((N, K)) * 0.04).astype(np.float32)
    g = (1.0 + 0.3 * rng.standard_normal(K)).astype(np.float32)
    b = (0.2 * rng.standard_normal(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    w_out, cvec = rt.debug_fold_ln(w, g, b, bias)
    KR.check_fold_ln("fold_ln", w_out, cvec, w, g, b, bias)


def _vit_embed_inputs(rng, T, n_items):
    patch = (rng.standard_normal((n_items * T, KR.H)) * 0.7 + 0.2).astype(np.float16)
    cls = rng.standard_normal(KR.H).astype(np.float32)
    pos = (0.5 * rng.standard_normal((T, KR.H))).astype(np.float32)
    g = (1.0 + 0.3 * rng.standard_normal(KR.H)).astype(np.float32)
    b = (0.2 * rng.standard_normal(KR.H)).astype(np.float32)
    return patch, cls, pos, g, b


@gpu
@pytest.mark.parametrize("T", [2, 197, 257])
def test_vit_embed(rt, T):
    rng = np.random.default_rng(T)
    args = _vit_embed_inputs(rng, T, 3)
    hi, lo, st = rt.debug_vit_embed(*args, T=T, eps=1e-5)
    KR.check_vit_embed(f"vit_embed T={T}", hi, lo, st, *args, T, 1e-5)


def _stream_rows(rng, rows, mean=0.0):
    x = (rng.standard_normal((rows, KR.H)) * 1.5 + mean).astype(np.float32)
    return KR.split_hilo(x)


@gpu
@pytest.mark.parametrize("S,n_items", [(1, 5), (7, 133), (512, 9)])
def test_pool_normalize(rt, S, n_items):
    """The CLS row of every item (row i * S), 133 items = not a multiple of the 8 warps per block; then a constant CLS row
    with beta = 0 gives an all-zero, finite vector, as F.normalize does."""
    rng = np.random.default_rng(S)
    hi, lo = _stream_rows(rng, n_items * S, mean=0.4)
    g = (1.0 + 0.3 * rng.standard_normal(KR.H)).astype(np.float32)
    b = (0.2 * rng.standard_normal(KR.H)).astype(np.float32)
    out = rt.debug_pool_normalize(hi, lo, g, b, S, 1e-12)
    KR.check_pool_normalize(f"pool_normalize S={S} n={n_items}", out, hi, lo, g, b, S, 1e-12)
    hi[0], lo[0] = np.float16(3.25), np.float16(2.0 ** -12)  # the row sums to exactly 768 x its value
    out = rt.debug_pool_normalize(hi, lo, g, np.zeros(KR.H, np.float32), S, 1e-12)
    assert np.isfinite(out).all() and (out[0] == 0.0).all(), out[0][:8]


@gpu
@pytest.mark.parametrize("P", [1, 7, 512, 1000, 1024])
def test_vit_pool(rt, P):
    T, n_items = 197, 5
    rng = np.random.default_rng(P)
    hi, lo = _stream_rows(rng, n_items * T, mean=-0.3)
    g = (1.0 + 0.3 * rng.standard_normal(KR.H)).astype(np.float32)
    b = (0.2 * rng.standard_normal(KR.H)).astype(np.float32)
    proj = (rng.standard_normal((P, KR.H)) * 0.03).astype(np.float32)
    out = rt.debug_vit_pool(hi, lo, g, b, proj, T, 1e-5)
    KR.check_vit_pool(f"vit_pool P={P}", out, hi, lo, g, b, proj, T, 1e-5)
    if P == 1024:
        with pytest.raises(rt.B200RTError) as e:
            rt.debug_vit_pool(hi, lo, g, b, np.zeros((1025, KR.H), np.float32), T, 1e-5)
        assert e.value.code == rt.E_INVALID
        rt.debug_vit_pool(hi, lo, g, b, proj, T, 1e-5)  # the rejected call left the runtime usable


# ================================================================================================ attention, exact answers

@gpu
def test_attention_single_key_returns_v0(rt):
    B, S = 3, 200
    rng = np.random.default_rng(8)
    qkv = (rng.standard_normal((B * S, 2304)) * 3.0).astype(np.float16)
    ctx, _ = rt.debug_attention(qkv, np.ones(B, np.int32), B, S)
    v0 = qkv.reshape(B, S, 2304)[:, :1, 1536:]
    same = np.array_equal(ctx.reshape(B, S, 768).view(np.uint16), np.broadcast_to(v0, (B, S, 768)).view(np.uint16))
    print(f"len 1: every query row equals V[0] bitwise: {same}")
    assert same


@gpu
def test_attention_zero_queries_average_the_valid_values(rt):
    B, S, lens = 3, 300, [300, 129, 64]
    rng = np.random.default_rng(9)
    qkv = (rng.standard_normal((B * S, 2304)) * 2.0).astype(np.float16)
    qkv[:, :768] = 0.0
    ctx, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S)
    v = qkv.reshape(B, S, 2304)[..., 1536:].astype(np.float64)
    mean = np.concatenate([np.broadcast_to(v[b, :n].mean(0), (S, 768)) for b, n in enumerate(lens)])
    ref, tol = KR.attention_ref(qkv, lens, B, S)
    assert np.allclose(ref, mean, rtol=1e-12, atol=1e-12)
    KR.check("Q = 0: mean of the valid V rows", ctx, mean, tol)


@gpu
@pytest.mark.parametrize("S", [512, 511])
def test_attention_lens_on_every_sub_block_boundary(rt, S):
    lens = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 511, 512]  # 512 at S = 511 is clamped to 511
    B = len(lens)
    rng = np.random.default_rng(S)
    qkv = (rng.standard_normal((B * S, 2304)) * 2.0).astype(np.float16)
    ctx, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S)
    KR.check_attention(f"lens on sub-block boundaries, S={S}", ctx, qkv, lens, B, S)


# ================================================================================================ CPU: the checks discriminate

GEMM_MUTANTS = {0: ["drop_kblock", "swap_halves", "permute_fragments", "bias_shift"],
                1: ["drop_kblock", "swap_halves", "permute_fragments", "bias_shift", "gelu_swap"],
                2: ["drop_kblock", "swap_halves", "permute_fragments", "bias_shift", "lo_dropped"],
                3: ["drop_kblock", "swap_halves", "permute_fragments", "bias_shift", "gelu_swap"]}


@pytest.mark.parametrize("epi,N,K", [(0, 512, 192), (1, 512, 192), (2, 512, 192), (3, 512, 192),  # plain epilogues
                                     (1, 256, 768), (3, 256, 768), (2, 768, 128)])                   # with the LayerNorm
def test_gemm_check_accepts_emulation_and_rejects_mutants(epi, N, K):
    args, kw = _gemm_case(epi, 256, N, K, seed=epi)
    if epi == 2:  # a residual large enough that dropping lo is far outside the hi + lo bound
        kw["resid"] = kw["resid"] * np.float32(30.0)
        if "ln_stats" in kw:
            kw["ln_stats"] = KR.partials(KR.hilo64(*KR.split_hilo(kw["resid"]))).astype(np.float32)
    KR.check_gemm(f"epi {epi} emulation", KE.emulate_gemm(epi, *args, **kw), epi, *args, **kw)
    for m in GEMM_MUTANTS[epi]:
        with pytest.raises(AssertionError):
            KR.check_gemm(f"epi {epi} mutant {m}", KE.emulate_gemm(epi, *args, mutant=m, **kw), epi, *args, **kw)


def test_gemm_stats_check_rejects_a_partial_about_the_row_mean():
    args, kw = _gemm_case(2, 128, 768, 128, seed=3, ln=False)
    v = KE.emulate_gemm(2, *args, **kw).astype(np.float64)
    sl = v.reshape(v.shape[0], -1, 128)
    good = np.stack([sl.sum(-1), ((sl - sl.mean(-1, keepdims=True)) ** 2).sum(-1)], -1).astype(np.float32)
    bad = np.stack([sl.sum(-1), ((sl - v.mean(-1)[:, None, None]) ** 2).sum(-1)], -1).astype(np.float32)
    KR.check_gemm_stats("stats emulation", good, args, **kw)
    with pytest.raises(AssertionError):
        KR.check_gemm_stats("stats mutant: row mean", bad, args, **kw)


def test_attention_check_accepts_emulation_and_rejects_mutants():
    """Scores that climb by sub-block (as in test_attention_running_max_rescale), lens short of S so that the key mask can be
    off by one in either direction."""
    B, S, lens = 2, 192, [150, 100]
    rng = np.random.default_rng(1)
    x = rng.standard_normal((B, S, 3, 12, 64)) * 0.5
    u = rng.standard_normal(64)
    u /= np.linalg.norm(u)
    x[:, :, 0] += 4.0 * np.where(rng.random((B, S, 12, 1)) < 0.6, 1.0, -1.0) * u
    x[:, :, 1] += (12.0 * (np.arange(S) // 64))[None, :, None, None] * u
    qkv = x.reshape(B * S, 2304).astype(np.float16)
    KR.check_attention("attention emulation", KE.emulate_attention(qkv, lens, B, S), qkv, lens, B, S)
    for m in ("mask_plus", "mask_minus", "no_rescale"):
        with pytest.raises(AssertionError):
            KR.check_attention(f"attention mutant {m}", KE.emulate_attention(qkv, lens, B, S, m), qkv, lens, B, S)


def test_row_checks_accept_emulations_and_reject_mutants():
    rng = np.random.default_rng(2)
    # embed: the bit-exact model itself, its fp32 partials, and three mutants
    vocab, S = 16, 40
    word, pos, type0 = _embed_tables(rng, vocab, S)
    ids = rng.integers(0, vocab, size=2 * S).astype(np.int32)
    hi, lo, x = KR.embed_exact(ids, word, pos, type0, S)
    KR.check_embed("embed emulation", hi, lo, KE.partials32(x), ids, word, pos, type0, S)
    hi_p, lo_p, x_p = KR.embed_exact(ids, word, np.roll(pos, -1, axis=0), type0, S)  # position t + 1
    with pytest.raises(AssertionError):
        KR.check_embed("embed mutant: position off by one", hi_p, lo_p, KE.partials32(x_p), ids, word, pos, type0, S)
    with pytest.raises(AssertionError):
        KR.check_embed("embed mutant: lo dropped", hi, np.zeros_like(lo), KE.partials32(x), ids, word, pos, type0, S)
    fin = np.isfinite(x).all(-1)
    with pytest.raises(AssertionError):
        KR.check_partials("embed mutant: partials about the row mean", KE.partials32(x[fin], True), x[fin].astype(np.float64))
    # vit_embed
    T = 197
    patch, cls, vpos, g, b = _vit_embed_inputs(rng, T, 2)
    tk = np.arange(patch.shape[0]) % T

    def vit_emul(shift):
        src = np.where((tk == 0)[:, None], cls[None, :], patch.astype(np.float32))
        y = KE.ln32(src + vpos[(tk + shift) % T], g, b, 1e-5)
        return (*KR.split_hilo(y), KE.partials32(y))

    KR.check_vit_embed("vit_embed emulation", *vit_emul(0), patch, cls, vpos, g, b, T, 1e-5)
    with pytest.raises(AssertionError):
        KR.check_vit_embed("vit_embed mutant: position off by one", *vit_emul(1), patch, cls, vpos, g, b, T, 1e-5)
    # pool_normalize / vit_pool: the wrong pooled row
    S = 7
    hi, lo = _stream_rows(rng, 9 * S, mean=0.4)
    x = hi.astype(np.float32) + lo.astype(np.float32)
    proj = (rng.standard_normal((64, KR.H)) * 0.03).astype(np.float32)

    def pooled(row0, P=None):
        z = KE.ln32(x[row0::S], g, b, 1e-12)
        if P is not None:
            z = z @ P.T
        return z / np.maximum(np.linalg.norm(z, axis=-1, keepdims=True), np.float32(1e-12))

    KR.check_pool_normalize("pool_normalize emulation", pooled(0), hi, lo, g, b, S, 1e-12)
    KR.check_vit_pool("vit_pool emulation", pooled(0, proj), hi, lo, g, b, proj, S, 1e-12)
    with pytest.raises(AssertionError):
        KR.check_pool_normalize("pool_normalize mutant: row 1", pooled(1), hi, lo, g, b, S, 1e-12)
    with pytest.raises(AssertionError):
        KR.check_vit_pool("vit_pool mutant: row 1", pooled(1, proj), hi, lo, g, b, proj, S, 1e-12)
    # fold_ln: an fp32 emulation passes
    w = (rng.standard_normal((40, 256)) * 0.04).astype(np.float32)
    wg = w * g[:256]
    cv = (w @ b[:256]).astype(np.float32)
    KR.check_fold_ln("fold_ln emulation", (wg - wg.mean(1, keepdims=True, dtype=np.float32)).astype(np.float16), cv, w, g[:256], b[:256], None)
