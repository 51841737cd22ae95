"""The GEMM's 2-CTA clusters: the two CTAs of a cluster take the two m-tiles of a tile pair, share its W tile by TMA
multicast and free each ring stage in both CTAs.  What that adds over an unclustered walk, each against the fp64 references
of tests/kernel_refs.py at their tolerances:

  * a pair whose second m-tile lies partly or wholly past M (an odd number of m-tiles), on one cluster that still has more
    pairs to walk and on every SM, for every epilogue, at both tile widths;
  * many pairs per cluster, so that the ring phases of both CTAs cross tile boundaries in step;
  * launch widths that are not whole clusters, and the split-SM runtime at an odd SM split.
"""
import numpy as np
import pytest

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
    return x.view(np.uint32 if x.dtype == np.float32 else np.uint16)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


# (epi, N, K, stats_out): every epilogue at BN = 256 (N = 768) and BN = 128 (N = 384), the residual one with and without
# the row statistics of its output
EPILOGUES = [(e, n, n, st) for n in (768, 384) for e, st in ((0, False), (1, False), (3, False), (2, True), (2, False))]


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
