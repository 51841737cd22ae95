"""The GEMM's 2-CTA clusters: the two CTAs of a cluster take the two m-tiles of a tile pair, share its W tile by TMA
multicast and free each ring stage in both CTAs.  What that adds over an unclustered walk, each against the fp64 references
of tests/kernel_refs.py at their tolerances:

  * a pair whose second m-tile lies partly or wholly past M (an odd number of m-tiles), on one cluster that still has more
    pairs to walk and on every SM, for every epilogue, at both tile widths;
  * many pairs per cluster, so that the ring phases of both CTAs cross tile boundaries in step;
  * launch widths that are not whole clusters, and the split-SM runtime at an odd SM split.

The same three for the epilogues nomic-bert and SPLADE added -- the rotary QKV GEMM (tests/nomic_refs.rope_gemm_ref), the
SwiGLU FFN1 GEMM (nomic_refs.swiglu_gemm_ref) and the SPLADE vocabulary max (tests/splade_refs.check_gemm_splade) -- with the
split runtime's GEMM widths among the launch widths: SPLIT_SMS(k) gives GEMMs 132 - k SMs (21: 111, 66: 66) and attention k.
Their debug entries report the CTAs they launched, so each case asserts the cluster shape it sets out to test.
"""
import numpy as np
import pytest

import kernel_refs as KR
import nomic_refs as NR
import splade_refs as SR

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _ln_inputs(rng, M, W, mean=0.3, std=1.7):
    y = (rng.standard_normal((M, W)) * std + mean).astype(np.float32)
    y += np.repeat(rng.standard_normal(W // 64) * 0.5, 64)[None, :].astype(np.float32)
    g = (1.0 + 0.3 * rng.standard_normal(W)).astype(np.float32)
    b = (0.2 * rng.standard_normal(W)).astype(np.float32)
    return y, g, b


def _gemm_case(epi, M, N, K, seed):
    """epi 0/1/3 fold a LayerNorm of the (K wide) A rows, epi 2 re-applies one to the (N wide) residual; that width is 768
    or 384.  Returns (args, kwargs) for both debug_gemm and kernel_refs.gemm_ref."""
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    kw = dict(eps=1e-12)
    if epi == 2:
        a = rng.standard_normal((M, K)).astype(np.float16)
        resid, g, b = _ln_inputs(rng, M, N, mean=-0.5, std=2.0)
        kw.update(resid=resid, ln_stats=KR.partials(KR.hilo64(*KR.split_hilo(resid))).astype(np.float32), ln_gamma=g, ln_beta=b)
    else:
        y, _, _ = _ln_inputs(rng, M, K)
        a = y.astype(np.float16)
        w = (w.astype(np.float32) - w.astype(np.float32).mean(1, keepdims=True)).astype(np.float16)
        kw["ln_stats"] = KR.partials(y).astype(np.float32)
    return (a, w, bias), kw


def _run(rt, epi, args, kw, want_stats, sms=0):
    r = rt.debug_gemm(epi, *args, want_stats=want_stats, sms=sms, want_ctas=True, **kw)
    return r[0], (r[2] if want_stats else None), r[-1]


def _bits(x):
    return x.view(np.uint16 if x.dtype == np.float16 else np.uint32)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


# (epi, N, K, stats_out): every epilogue at BN = 256 (N = 768) and BN = 128 (N = 384), the residual one with and without
# the row statistics of its output; then the folded epilogues' other pairings of tile width and partials: BN = 128 with a
# 768-wide LayerNorm (6 partials) and BN = 256 with a 384-wide one (3 partials)
EPILOGUES = ([(e, n, n, st) for n in (768, 384) for e, st in ((0, False), (1, False), (3, False), (2, True), (2, False))]
             + [(e, 384, 768, False) for e in (0, 1, 3)] + [(e, 768, 384, False) for e in (0, 1, 3)])


@gpu
@pytest.mark.parametrize("M", [1, 129, 257, 8320])  # 1, 2, 3 and 65 m-tiles: the last pair's second tile past M
@pytest.mark.parametrize("epi,N,K,stats", EPILOGUES)
def test_partner_tile_past_m(rt, epi, N, K, stats, M):
    """On one cluster (sms = 2), which walks every pair -- the partial one included -- and on every SM: each against the
    fp64 reference, and the two bitwise equal."""
    args, kw = _gemm_case(epi, M, N, K, seed=M + 10 * epi + N + stats)
    tag = f"epi {epi} N={N} M={M}{' stats_out' if stats else ''}"
    one, one_st, ctas = _run(rt, epi, args, kw, stats, sms=2)
    assert ctas == 2, ctas
    KR.check_gemm(f"{tag} sms 2", one, epi, *args, **kw)
    if stats:
        KR.check_gemm_stats(f"{tag} sms 2: stats_out", one_st, args, **kw)
    every, every_st, _ = _run(rt, epi, args, kw, stats)
    same = _same(every, one) and (not stats or _same(every_st, one_st))
    print(f"{tag}: sms 2 within tolerance, bitwise equal to every SM: {same}")
    assert same


@gpu
@pytest.mark.parametrize("epi,N,K", [(1, 3072, 768), (2, 768, 3072)])  # bge-base FFN1 (12 k-blocks), FFN2 (48 k-blocks)
def test_many_pairs_per_cluster(rt, epi, N, K):
    """M = 4096: 32 m-tiles, 192 / 48 tile pairs, all walked by one cluster, whose 4-stage rings wrap 576 times in step;
    bitwise equal to the launch on every SM."""
    M = 4096
    args, kw = _gemm_case(epi, M, N, K, seed=40 + epi)
    want = epi == 2
    base, base_st, ctas = _run(rt, epi, args, kw, want)
    assert ctas % 2 == 0 and ctas > 2, ctas
    KR.check_gemm(f"epi {epi} N={N} K={K} every SM ({ctas} CTAs)", base, epi, *args, **kw)
    one, one_st, _ = _run(rt, epi, args, kw, want, sms=2)
    same = _same(one, base) and (not want or _same(one_st, base_st))
    print(f"epi {epi} N={N} K={K}: one cluster bitwise equal to {ctas} CTAs: {same}")
    assert same


@gpu
@pytest.mark.parametrize("epi,N,K", [(0, 2304, 768), (2, 768, 768), (0, 1152, 384)])
def test_widths_that_are_not_whole_clusters(rt, epi, N, K):
    """sms = 1, 3, 131 launch 2, 2 and at most 130 CTAs (whole clusters, at least one), bitwise equal to every SM."""
    M = 4100
    args, kw = _gemm_case(epi, M, N, K, seed=50 + epi + N)
    want = epi == 2
    base, base_st, _ = _run(rt, epi, args, kw, want)
    KR.check_gemm(f"epi {epi} N={N} every SM", base, epi, *args, **kw)
    for sms in (1, 3, 131):
        got, got_st, ctas = _run(rt, epi, args, kw, want, sms=sms)
        assert ctas % 2 == 0 and 2 <= ctas <= max(2, sms), (sms, ctas)
        same = _same(got, base) and (not want or _same(got_st, base_st))
        print(f"epi {epi} N={N}: sms {sms} -> {ctas} CTAs, bitwise equal to every SM: {same}")
        assert same, sms


@gpu
def test_split_sm_runtime_odd_split(rt):
    """B200RT_INIT_SPLIT_SMS(21): the GEMMs get 111 SMs, i.e. 55 clusters; a ragged text batch spread over both replicas
    gives the whole-GPU runtime's bits.  The module's runtime is shut down for the duration and restarted afterwards."""
    from oracle import bge_ref as R

    tg = R.BertGeometry(layers=2)
    tblob = R.pack_blob(R.make_weights(tg, 3, "trained"), tg)
    ids, lens = R.synth_ragged(40, 512, seed=13, min_len=1)

    def run(flags):
        rt.shutdown()
        rt.init(devices=[0], flags=flags)
        out = rt.EmbedModel(R.geometry_dict(tg), tblob).embed(ids, lens)
        return out, rt.num_gpus(), rt.stats()["peer_bytes"]

    try:
        whole, n_whole, _ = run(0)
        split, n_split, peer = run(rt.SPLIT_SMS(21))
    finally:
        rt.shutdown()
        rt.init(devices=[0])
    assert n_whole == 1 and n_split == 2
    assert peer > 0, "the second replica took no items"
    same = np.array_equal(whole.view(np.uint32), split.view(np.uint32))
    print(f"split SMs k=21: ragged text ({whole.shape[0]} items) bitwise equal to the whole-GPU runtime: {same}")
    assert same


# ------------------------------------------------------------------------------------------------ rotary, SwiGLU, SPLADE
#
# Each case is (run, check): run(rt, sms) -> (out, ctas) through the debug entry, check(tag, out) -> the worst err/tol against
# the fp64 reference at its tolerance.

def _nomic_stats(rng, M):
    """(sum, M2) partials of random 768-wide rows of mean ~0.3, sd ~1.5."""
    return KR.partials(rng.standard_normal((M, 768)) * 1.5 + 0.3).astype(np.float32)


def _rope_case(M, S, ln, seed):
    """QKV of nomic-bert: N = 2304, the first rot_cols = 1536 columns (Q and K) rotated by position row % S, V not."""
    rng = np.random.default_rng(seed)
    a = (rng.standard_normal((M, 768)) * 1.2).astype(np.float16)
    w = (rng.standard_normal((2304, 768)) * 0.05).astype(np.float16)
    c = (rng.standard_normal(2304) * 0.1).astype(np.float32)
    st = _nomic_stats(rng, M) if ln else None
    table = NR.rope_table(S, 1000.0)

    def run(rt, sms):
        return rt.debug_gemm_rope(a, w, c, st, table, S, 1536, 1e-12, sms=sms, want_ctas=True)

    def check(tag, out):
        ref, tol = NR.rope_gemm_ref(a, w, c, st, table, S, 1536, 1e-12, pos=np.arange(M) % S)
        return KR.check(tag, out.astype(np.float64), ref, tol)
    return run, check


def _swiglu_case(M, ln, seed):
    """FFN1 of nomic-bert: gate and up (3072 rows each) interleaved in groups of 8, N = 6144, out [M, 3072]."""
    rng = np.random.default_rng(seed)
    a = (rng.standard_normal((M, 768)) * 1.2).astype(np.float16)
    w = NR.interleave_rows(rng.standard_normal((3072, 768)) * 0.05, rng.standard_normal((3072, 768)) * 0.05).astype(np.float16)
    c = (NR.interleave_rows(rng.standard_normal((3072, 1)), rng.standard_normal((3072, 1)))[:, 0] * 0.3).astype(np.float32)
    st = _nomic_stats(rng, M) if ln else None

    def run(rt, sms):
        return rt.debug_gemm_swiglu(a, w, c, st, 1e-12, sms=sms, want_ctas=True)

    def check(tag, out):
        ref, tol = NR.swiglu_gemm_ref(a, w, c, st, 1e-12)
        return KR.check(tag, out.astype(np.float64), ref, tol)
    return run, check


def _splade_lens(B, S, rng):
    """Ragged lengths: S, 1, the 63 / 64 / 65 edges (65 clamps to S when S = 64), S - 1, then random."""
    edges = np.array([S, 1, 63, 64, 65, S - 1], np.int32)
    return np.concatenate([edges, rng.integers(1, S + 1, max(0, B - len(edges)))]).astype(np.int32)[:B]


def _splade_case(B, S, K, vocab, seed):
    """The decoder GEMM of B items of S rows: K = 384 / 768 / 1024 (PARTS 3 / 6 / 8), N = vocab tiled to 256.  Operands as
    tests/test_gpu_splade.py's: ~60 % of the logits positive, a fifth of the columns' c so negative that they stay 0."""
    rng = np.random.default_rng(seed)
    lens = _splade_lens(B, S, rng)
    x = rng.standard_normal((B * S, K))
    u = (x * (x > -0.5) * 1.3 + 0.2 * rng.standard_normal(K)).astype(np.float16)
    stats = KR.partials(u.astype(np.float64)).astype(np.float32)
    w = (rng.standard_normal((vocab, K)) * (1.0 / np.sqrt(K))).astype(np.float16)
    N = SR.vpad(vocab)
    c = (rng.standard_normal(N) - 1.0).astype(np.float32)
    c[rng.random(N) < 0.2] = -20.0

    def run(rt, sms):
        out, _, ctas = rt.debug_gemm_splade(u, w, c, stats, lens, S, N, 1e-12, sms=sms, want_ctas=True)
        return out, ctas

    def check(tag, out):
        return SR.check_gemm_splade(tag, out, u, w, c, stats, lens, S, 1e-12)
    return run, check


def _bm_tiles(M):
    return (M + 127) // 128


# rotary: M = B S with an odd m-tile count or a partial last tile.  S = 64 puts two items in a 128-row tile; S = 192 never
# splits a 64-row half across items.  M = 64, 192, 576 and 8256 (1, 2 -- the second partial --, 5 and 65 m-tiles).
ROPE_PAST_M = [(B, S) for S, Bs in ((64, (1, 3, 129)), (192, (1, 3, 43))) for B in Bs]
# SPLADE: (B, S, vocab).  30522 words (the last 256-column tile partial) at S = 64; elsewhere a narrower vocabulary, still
# ending in a partial tile, keeps the fp64 reference's [B S, vocab] logits small.
SPLADE_PAST_M = [(1, 64, 30522), (3, 64, 30522), (129, 64, 2000), (3, 192, 2000)]


def _past_m(rt, tag, run, check):
    one, ctas = run(rt, 2)
    assert ctas == 2, ctas
    margin = check(f"{tag} sms 2", one)
    every, _ = run(rt, 0)
    same = _same(every, one)
    print(f"{tag}: sms 2 (worst err/tol {margin:.3f}) bitwise equal to every SM: {same}")
    assert same


@gpu
@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("B,S", ROPE_PAST_M)
def test_rope_partner_tile_past_m(rt, B, S, ln):
    M = B * S
    run, check = _rope_case(M, S, ln, seed=M + S + ln)
    _past_m(rt, f"rope M={M} S={S} ({_bm_tiles(M)} m-tiles) ln={ln}", run, check)


@gpu
@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("M", [1, 129, 257, 8320])
def test_swiglu_partner_tile_past_m(rt, M, ln):
    run, check = _swiglu_case(M, ln, seed=M + 7 * ln)
    _past_m(rt, f"swiglu M={M} ({_bm_tiles(M)} m-tiles) ln={ln}", run, check)


SPLADE_KS = [384, 768, 1024]  # PARTS 3, 6, 8


@gpu
@pytest.mark.parametrize("K", SPLADE_KS)
@pytest.mark.parametrize("B,S,vocab", SPLADE_PAST_M)
def test_splade_partner_tile_past_m(rt, B, S, vocab, K):
    """The maxima are an integer max of fp32 bits (order-independent), so any bitwise difference is a real bug."""
    run, check = _splade_case(B, S, K, vocab, seed=B * S + K)
    _past_m(rt, f"splade K={K} B={B} S={S} vocab={vocab} ({_bm_tiles(B * S)} m-tiles)", run, check)


# M = 4096: 16 m-tile pairs.  rotary: 9 n-tiles, 144 pairs; SwiGLU: 24 n-tiles, 384 pairs; SPLADE: 8 items of 512 (each over
# 4 m-tiles, so an item's maxima merge across tiles and both CTAs), vocabulary 4000 -> 16 n-tiles, 256 pairs.
NEW_EPILOGUES = {
    "rope": lambda M: _rope_case(M, 64 if M % 512 else 512, True, seed=M),
    "swiglu": lambda M: _swiglu_case(M, True, seed=M + 1),
    "splade": lambda M: _splade_case(M // 512 if M % 512 == 0 else M // 64, 512 if M % 512 == 0 else 64, 768, 4000, seed=M + 2),
}


@gpu
@pytest.mark.parametrize("epi", list(NEW_EPILOGUES))
def test_new_epilogues_many_pairs_per_cluster(rt, epi):
    """Every pair of M = 4096 walked by one cluster (sms = 2), bitwise the launch on every SM; the reference once, on every SM."""
    run, check = NEW_EPILOGUES[epi](4096)
    base, ctas = run(rt, 0)
    assert ctas % 2 == 0 and ctas > 2, ctas
    margin = check(f"{epi} M=4096 every SM ({ctas} CTAs)", base)
    one, one_ctas = run(rt, 2)
    assert one_ctas == 2, one_ctas
    same = _same(one, base)
    print(f"{epi} M=4096: one cluster bitwise equal to {ctas} CTAs: {same} (worst err/tol {margin:.3f})")
    assert same


@gpu
@pytest.mark.parametrize("epi", list(NEW_EPILOGUES))
def test_new_epilogues_widths_that_are_not_whole_clusters(rt, epi):
    """sms = 1, 3, 131 (not whole clusters) and 21, 66, 111 (the split runtime's attention and GEMM widths), each bitwise the
    launch on every SM.  M = 4160 (33 m-tiles: the last pair's second tile past M); SPLADE: 65 items of 64."""
    run, check = NEW_EPILOGUES[epi](4160)
    base, base_ctas = run(rt, 0)
    check(f"{epi} M=4160 every SM ({base_ctas} CTAs)", base)
    for sms in (1, 3, 21, 66, 111, 131):
        got, ctas = run(rt, sms)
        assert ctas % 2 == 0 and 2 <= ctas <= max(2, sms), (sms, ctas)
        same = _same(got, base)
        print(f"{epi} M=4160: sms {sms} -> {ctas} CTAs, bitwise equal to every SM: {same}")
        assert same, sms
