"""Forward-chain conformance at full wave size: every launch of each model's production-size forward against its fp64 reference.

tests/test_gpu_forward_chain.py checks every launch of the forward on a toy wave (at most a few thousand rows).  The product
runs waves 30-100x larger, and there the kernels take other paths: dozens of GEMM tiles per 2-CTA cluster, attention unsplit
with many (item, head) units per CTA, plain launches instead of graph replay.  Here each model runs one wave at its full
capacity (`debug_cap_rows() // S` items, so a card with fewer SMs gets its own full wave) and `run_chain` checks every launch.

An fp64 reference of every row is too expensive on the host (about 2 TFLOP per bge-base layer), so the row-wise checks read a
sample chosen by `sample_rows`, every column of each sampled row:
  * GEMMs: one row in each 64-row consumer half of each 128-row m-tile.  The row's offset in its half walks the 64 offsets with
    stride 37 from tile to tile, so across a wave every 16-row warp slice and both fragment rows (r, r + 8) are read;
  * attention: one query row in each (item, 128-row query tile, 64-row warpgroup half), padding rows included; with every
    column read, that is each head of each such block;
  * all rows of the first and the last item;
  * the residual epilogues' `stats_out` partials and the embedding's partials on the same rows.
A wrong tile, a swapped half, a stale or foreign statistics tile or a misrouted attention block is therefore always read.  The
cheap checks stay whole: embed / im2col bit for bit and vit_embed over every row, every pool over every item (mean pooling
over every valid row), and run_chain's buffer invariants over the whole buffers.

Each GPU case prints its worst err / tol per launch and then asserts that embed_device (text models) and the scheduler's
embed() of the same wave are bitwise the traced pooled output, the path bench.py times.  The CPU tests run the same sampled
checks on a numpy emulation of a reduced wave (bge-base widths, B = 8 at S = 256): they accept it, they reject every
corruption above at every position, the wiring mutants of tests/test_gpu_forward_chain.py are still caught, the subset
attention references equal the full ones on their rows, and the sampling rule covers each GPU case's real shape."""
import resource
import time

import numpy as np
import pytest

import attention_refs as AR
import clip_text_refs as T
import kernel_emul as KE
import kernel_refs as KR
import test_gpu_clip_text as CT
import test_gpu_forward_chain as FC
from oracle import bge_ref as R
from oracle import clip_ref as C

gpu = pytest.mark.gpu

BM, HALF, QT = 128, 64, 128  # GEMM m-tile rows (two consumer halves), attention query-tile rows (two warpgroup halves)
STRIDE = 37                  # odd, so the offsets of 64 successive tiles are all 64 rows of a half


def _offset(j, h, n):
    """Sampled row within a half of n rows: half h of tile (or query tile) j."""
    return (STRIDE * j + 23 * h) % n


def sample_rows(B, S):
    """Ascending rows of a B x S wave the row-wise checks read (see the module docstring)."""
    M = B * S
    picks = [np.arange(S), np.arange(M - S, M)]
    gemm = [t * BM + h * HALF + _offset(t, h, min(HALF, M - t * BM - h * HALF))
            for t in range(-(-M // BM)) for h in (0, 1) if t * BM + h * HALF < M]
    nq = -(-S // QT)
    attn = [b * S + q * QT + h * HALF + _offset(b * nq + q, h, min(HALF, S - q * QT - h * HALF))
            for b in range(B) for q in range(nq) for h in (0, 1) if q * QT + h * HALF < S]
    return np.unique(np.concatenate(picks + [np.asarray(gemm, np.int64), np.asarray(attn, np.int64)]))


def coverage(rows, B, S):
    """Asserts what sample_rows promises for a B x S wave; returns a one-line summary."""
    M = B * S
    rows = np.asarray(rows)
    assert np.array_equal(np.unique(rows // HALF), np.arange(-(-M // HALF))), "a GEMM (m-tile, half) without a sampled row"
    middle = rows[(rows >= S) & (rows < M - S)]  # what the rule itself picks, outside the items read whole
    for h in (0, 1):
        off = middle[(middle // HALF) % 2 == h] % HALF
        assert len(set(off.tolist())) == HALF, f"half {h}: sampled offsets miss rows of a warp slice / fragment"
    w = rows % S
    blocks = set(zip((rows // S).tolist(), (w // HALF).tolist()))
    assert len(blocks) == B * -(-S // HALF), "an (item, query tile, half) without a sampled query row"
    assert np.isin(np.r_[0:S, M - S:M], rows).all(), "the first and last items are not read whole"
    return f"{B} x {S}: {len(rows)} of {M} rows sampled"


def wave_shapes(rt_rows):
    """(B, S) of each GPU case for a runtime of rt_rows workspace rows (512 per SM): bge-large holds 3/4 of them, rounded down
    to 128 (tests/test_bge_large.py spec_cap_rows)."""
    large = rt_rows * 768 // 1024 // BM * BM
    return {"base": (rt_rows // 512, 512), "small_mean": (rt_rows // 512, 512), "large": (large // 512, 512),
            "clip_text_128": (rt_rows // 128, 128), "clip_text_64": (rt_rows // 64, 64), "vit": (64, 197)}


def ragged_lens(B, S, seed, max_len=None):
    """Seeded lengths over [1, max_len] (default S), with 1, max_len and both sides of every 64-key sub-block edge among them."""
    L = max_len or S
    edges = [1, L] + [e for k in range(64, L + 1, 64) for e in (k - 1, k, k + 1) if e <= L]
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, L + 1, B)
    lens[rng.permutation(B)[:len(edges)]] = edges[:B]
    return lens.astype(np.int32)


# ================================================================================================ GPU

_T0 = time.perf_counter()


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()
    print(f"\ntest_gpu_full_wave_chain: {time.perf_counter() - _T0:.1f} s wall time, "
          f"peak RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20:.2f} GB")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _device_embed(rt, model, ids, lens, out_dim):
    """embed_device of the whole wave on replica 0 (plain launches, device-resident ids and output)."""
    import torch

    d_ids, d_lens = torch.from_numpy(np.ascontiguousarray(ids)).cuda(), torch.from_numpy(np.ascontiguousarray(lens)).cuda()
    d_out = torch.empty((ids.shape[0], out_dim), dtype=torch.float32, device="cuda")
    model.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), ids.shape[0], ids.shape[1], d_out.data_ptr(), 0)
    rt.device_sync(0)
    return d_out.cpu().numpy()


TEXT = {"base": (dict(), "cls"), "small_mean": (dict(hidden=384, heads=12, inter=1536), "mean"),
        "large": (dict(hidden=1024, heads=16, inter=4096), "cls")}


def _run(tag, ch, trace, cap_rows, t0):
    margins = {}
    last = FC.run_chain(tag, ch, trace, margins, cap_rows=cap_rows)
    FC.print_margins(f"{tag} ({ch.B} x {ch.S}, {len(ch.rows)} of {ch.M} rows sampled)", margins)
    print(f"{tag}: chain checked in {time.perf_counter() - t0:.1f} s")
    assert max(margins.values()) < 1
    return last


@gpu
@pytest.mark.parametrize("case", list(TEXT))
def test_text_full_wave_chain(rt, case):
    t0 = time.perf_counter()
    geom, pooling = TEXT[case]
    g = R.BertGeometry(layers=2, **geom)
    flat = R.make_weights(g, 3, "trained")
    model = rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g), pooling=pooling)
    cap = model.debug_cap_rows()
    B, S = cap // 512, 512
    ids, lens = FC.ragged_batch(ragged_lens(B, S, seed=len(case)), S, seed=41)
    ch = FC.TextChain(flat, g, ids, lens, FC.gpu_fold(rt), rows=sample_rows(B, S))
    print(f"\n{case}: {coverage(ch.rows, B, S)}, {int((ch.rows % S >= lens[ch.rows // S]).sum())} of them padding")
    last = _run(case, ch, lambda k: model.debug_trace(ids, lens, k), cap, t0)
    assert last["n_total"] == 5 * g.layers + 2 and last["names"][-1] == ("mean_pool_normalize" if pooling == "mean" else "pool_normalize")
    assert np.array_equal(_bits(_device_embed(rt, model, ids, lens, g.hidden)), _bits(last["out"])), "embed_device differs from the trace"
    assert np.array_equal(_bits(model.embed(ids, lens)), _bits(last["out"])), "embed() differs from the traced pooled output"


@gpu
@pytest.mark.parametrize("S,max_len", [(128, 77), (64, 64)])
def test_clip_text_full_wave_chain(rt, S, max_len):
    t0 = time.perf_counter()
    g = T.geometry(layers=2, eos_id=T.EOS)
    flat = T.make_weights(g, 1, "trained")
    model = rt.ClipTextModel(g, T.pack_blob(flat, g))
    cap = model.debug_cap_rows()
    B = cap // S
    lens = ragged_lens(B, S, seed=S, max_len=max_len)
    ids = T.synth_ids(lens, S, seed=5)
    ch = CT.ClipTextChain(flat, g, ids, lens, FC.gpu_fold(rt), rows=sample_rows(B, S))
    print(f"\nclip_text {S}: {coverage(ch.rows, B, S)}")
    last = _run(f"clip_text {S}", ch, lambda k: model.debug_trace(ids, lens, k), cap, t0)
    assert last["n_total"] == 5 * g["layers"] + 2 and last["names"][-1] == "clip_text_pool"
    assert np.array_equal(_bits(_device_embed(rt, model, ids, lens, g["proj"])), _bits(last["out"])), "embed_device differs"
    assert np.array_equal(_bits(model.embed(ids[:, :max_len], lens)), _bits(last["out"])), "embed() differs from the trace"


@gpu
def test_vit_full_wave_chain(rt):
    t0 = time.perf_counter()
    g = C.VitGeometry(layers=2)
    flat = C.make_weights(g, 1, "trained")
    model = rt.ImageEmbedModel(C.geometry_dict(g), C.pack_blob(flat, g))
    B, S = wave_shapes(rt.wave_capacity_items() * 512)["vit"]
    px = C.synth_pixels(B, g, 4)
    ch = FC.VitChain(flat, g, px, FC.gpu_fold(rt), rows=sample_rows(B, S))
    print(f"\nvit: {coverage(ch.rows, B, S)}")
    last = _run("vit", ch, lambda k: model.debug_trace(px, k), rt.wave_capacity_items() * 512, t0)
    assert last["n_total"] == 5 * g.layers + 4 and last["rows"] == ch.M + FC.GUARD
    assert np.array_equal(_bits(model.embed(px)), _bits(last["out"])), "embed() differs from the traced pooled output"


# ================================================================================================ CPU: the sampled checks discriminate

CPU_LENS, CPU_S = [129, 1, 64, 65, 256, 127, 192, 63], 256


@pytest.fixture(scope="module")
def wave():
    """bge-base widths, 2 layers, `trained` weights, B = 8 at S = 256 (16 m-tiles), emulated; the chain samples its rows."""
    g = R.BertGeometry(layers=2)
    flat = R.make_weights(g, 3, "trained")
    ids, lens = FC.ragged_batch(CPU_LENS, CPU_S, seed=5)
    ch = FC.TextChain(flat, g, ids, lens, KE.fold_ln32, rows=sample_rows(len(CPU_LENS), CPU_S))
    return ch, FC.emulate_chain(ch)


def test_sampled_checks_accept_the_emulated_wave(wave):
    ch, traces = wave
    margins = {}
    FC.run_chain("emulated, sampled", ch, traces.__getitem__, margins)
    FC.print_margins("emulated, sampled", margins)
    # at capacity: no guard rows
    cut = [dict(t, **{b: t[b][:ch.M] for b in FC.BUFFERS}, rows=ch.M) for t in traces]
    FC.run_chain("emulated at capacity", ch, cut.__getitem__, cap_rows=ch.M)


def _launches(traces, names):
    """(k, layer, name) of the layer-1 launches named."""
    k0 = traces[-1]["names"].index("gemm_qkv", 2)
    return [(k, 1, traces[k]["names"][-1]) for k in range(k0 + 1, k0 + 6) if traces[k]["names"][-1] in names]


GEMM_OUT = {"gemm_qkv": ("qkv",), "gemm_attn_out": ("yhi", "ylo"), "gemm_ffn1_gelu": ("ffn",), "gemm_ffn2": ("yhi", "ylo")}
STATS_OUT = {"gemm_attn_out": "pstats1", "gemm_ffn2": "pstats0"}


def _feed(h, x):
    if isinstance(x, np.ndarray):
        h.update(repr((x.dtype.str, x.shape)).encode())
        h.update(np.ascontiguousarray(x).tobytes())
    elif isinstance(x, (list, tuple)):
        h.update(b"(")
        for y in x:
            _feed(h, y)
        h.update(b")")
    else:
        h.update(repr(x).encode())


@pytest.fixture
def memo_refs(monkeypatch):
    """The fp64 GEMM and attention references depend only on a launch's operands, which a corruption of its output leaves
    alone: each is computed once per distinct set of operands (keyed on their bytes), so that every position can be tried at
    the cost of the comparison alone."""
    import hashlib

    def memo(fn):
        cache = {}

        def wrapped(*args, **kw):
            h = hashlib.sha1()
            _feed(h, (args, sorted(kw.items())))
            k = h.digest()
            if k not in cache:
                cache[k] = fn(*args, **kw)
            return cache[k]
        return wrapped

    monkeypatch.setattr(KR, "gemm_ref", memo(KR.gemm_ref))
    monkeypatch.setattr(KR, "attention_ref", memo(KR.attention_ref))


def _rejects(ch, l, name, prev, cur, what):
    """The corruption keeps every buffer invariant (it stays inside the rows < M the launch writes, finite); the launch's
    sampled check must reject it."""
    FC.check_invariants(what, name, prev, cur, ch)
    with pytest.raises(AssertionError):
        ch.check(what, name, l, prev, cur)


def _tiles(ch):
    return -(-ch.M // BM)


def test_sampled_checks_reject_a_stale_or_foreign_gemm_tile(wave, memo_refs):
    """Every m-tile of each GEMM launch of layer 1 (the n-tile walks the columns): its 128 x 128 output tile holding the value
    the buffer had before the launch (stale), or the next m-tile's (foreign)."""
    ch, traces = wave
    n = 0
    for k, l, name in _launches(traces, GEMM_OUT):
        prev, cur = traces[k - 1], traces[k]
        for t in range(_tiles(ch)):
            buf = GEMM_OUT[name][0]
            c0 = (t % (cur[buf].shape[1] // 128)) * 128
            rs, cs = slice(t * BM, (t + 1) * BM), slice(c0, c0 + 128)
            ft = slice(((t + 1) % _tiles(ch)) * BM, ((t + 1) % _tiles(ch) + 1) * BM)
            for kind, src in (("stale", prev[buf][rs, cs]), ("foreign", cur[buf][ft, cs])):
                bad = dict(cur, **{buf: cur[buf].copy()})
                bad[buf][rs, cs] = src
                _rejects(ch, l, name, prev, bad, f"{name} m-tile {t} {kind}")
                n += 1
    print(f"{n} stale / foreign GEMM tiles rejected")


def test_sampled_checks_reject_swapped_halves(wave, memo_refs):
    """Every m-tile of each GEMM launch of layer 1: its two 64-row halves exchanged (every buffer the launch writes)."""
    ch, traces = wave
    n = 0
    for k, l, name in _launches(traces, GEMM_OUT):
        prev, cur = traces[k - 1], traces[k]
        for t in range(_tiles(ch)):
            bad = dict(cur)
            for buf in FC.WRITES[name]:
                x = cur[buf].copy()
                x[t * BM:(t + 1) * BM] = np.concatenate([x[t * BM + HALF:(t + 1) * BM], x[t * BM:t * BM + HALF]])
                bad[buf] = x
            _rejects(ch, l, name, prev, bad, f"{name} m-tile {t} halves swapped")
            n += 1
    print(f"{n} swapped m-tiles rejected")


def test_sampled_checks_reject_a_neighbours_stats_tile(wave, memo_refs):
    """Every m-tile of each residual epilogue of layer 1: its stats_out rows taken from the neighbouring m-tile."""
    ch, traces = wave
    n = 0
    for k, l, name in _launches(traces, STATS_OUT):
        prev, cur = traces[k - 1], traces[k]
        buf = STATS_OUT[name]
        for t in range(_tiles(ch)):
            u = t + 1 if t + 1 < _tiles(ch) else t - 1
            bad = dict(cur, **{buf: cur[buf].copy()})
            bad[buf][t * BM:(t + 1) * BM] = cur[buf][u * BM:(u + 1) * BM]
            _rejects(ch, l, name, prev, bad, f"{name} m-tile {t} {buf} from m-tile {u}")
            n += 1
    print(f"{n} neighbour statistics tiles rejected")


def test_sampled_checks_reject_a_misrouted_attention_block(wave, memo_refs):
    """Every (item, head, query tile, half) of layer 1's attention: that 64 x 64 block of ctx taken from the next item, or from
    the next head."""
    ch, traces = wave
    (k, l, name), = _launches(traces, ("attention",))
    prev, cur = traces[k - 1], traces[k]
    H, hd, S = ch.g.hidden, ch.hd, ch.S
    n = 0
    for b in range(ch.B):
        for head in range(ch.g.heads):
            for q in range(-(-S // QT)):
                for h in (0, 1):
                    r0 = b * S + q * QT + h * HALF
                    rs, cs = slice(r0, r0 + HALF), slice(head * hd, (head + 1) * hd)
                    ob = ((b + 1) % ch.B - b) * S
                    oc = slice(((head + 1) % ch.g.heads) * hd, ((head + 1) % ch.g.heads + 1) * hd)
                    for kind, src in (("item", cur["ctx"][r0 + ob:r0 + ob + HALF, cs]), ("head", cur["ctx"][rs, oc])):
                        bad = dict(cur, ctx=cur["ctx"].copy())
                        bad["ctx"][rs, cs] = src
                        _rejects(ch, l, name, prev, bad, f"attention item {b} head {head} tile {q} half {h} from the next {kind}")
                        n += 1
    print(f"{n} misrouted attention blocks rejected")


@pytest.mark.parametrize("mutant", FC.MUTANTS)
def test_sampled_checks_catch_the_wiring_mutants(wave, mutant):
    ch, _ = wave
    traces = FC.emulate_chain(ch, mutant)
    with pytest.raises(AssertionError) as e:
        FC.run_chain(f"mutant {mutant}, sampled", ch, traces.__getitem__)
    print(f"mutant {mutant}: caught: {str(e.value).splitlines()[0][:160]}")


def test_subset_attention_references_match_the_full_ones():
    rng = np.random.default_rng(3)
    S, lens = 192, [192, 1, 64, 65, 130]
    B = len(lens)
    rows = sample_rows(B, S)
    q_rows = [rows[(rows >= b * S) & (rows < (b + 1) * S)] - b * S for b in range(B)]
    for what, H, full, sub in (
            ("kernel_refs 12 x 64", 768, lambda x: KR.attention_ref(x, lens, B, S), lambda x: KR.attention_ref(x, lens, B, S, q_rows)),
            ("attention_refs 12 x 32", 384, lambda x: AR.attention_ref(x, lens, B, S, 12, 32),
             lambda x: AR.attention_ref(x, lens, B, S, 12, 32, q_rows)),
            ("attention_refs 16 x 64", 1024, lambda x: AR.attention_ref(x, lens, B, S, 16, 64),
             lambda x: AR.attention_ref(x, lens, B, S, 16, 64, q_rows)),
            ("causal 8 x 64", 512, lambda x: T.causal_attention_ref(x, lens, B, S), lambda x: T.causal_attention_ref(x, lens, B, S, rows=q_rows))):
        qkv = (rng.standard_normal((B * S, 3 * H)) * 1.5).astype(np.float16)
        (r0, t0), (r1, t1) = full(qkv), sub(qkv)
        assert r1.shape == (len(rows), H)
        np.testing.assert_allclose(r1, r0[rows], rtol=1e-12, atol=0, err_msg=what)
        np.testing.assert_allclose(t1, t0[rows], rtol=1e-12, atol=0, err_msg=what)
        print(f"{what}: {len(rows)} sampled query rows equal the full reference's")


@pytest.mark.parametrize("sms", [132, 114])
def test_sampling_covers_every_gpu_case(sms):
    for case, (B, S) in wave_shapes(sms * 512).items():
        print(f"{sms} SMs, {case}: {coverage(sample_rows(B, S), B, S)}")
