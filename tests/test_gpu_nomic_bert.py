"""GPU: nomic-bert (kind "nomic_bert") -- the three kernels the kind adds, the forward launch by launch, parity with the fp64
oracle up to 8192 tokens, and bitwise invariance of an item's embedding.

  * kernels through the debug entries against their fp64 references (tests/nomic_refs.py): the rotary QKV GEMM and the SwiGLU
    GEMM for M from 1 to past a 128-row tile at several S; the streaming attention for S in {64, 576, 1024, 2048, 4096, 8192}
    with lengths on every tile boundary, one valid key and Q = 0;
  * the streaming attention is bitwise the same at every launch width from 1 CTA to every SM (many units per CTA, and fewer
    units than CTAs), and bitwise attention_kernel<64, 12>'s for every S <= 512;
  * the forward launch by launch through run_chain (tests/test_gpu_forward_chain.py) with NomicChain, a TextChain for the
    kind's launches, on toy ragged batches and on a full wave of 8 x 8192 tokens (a row sample after
    tests/test_gpu_full_wave_chain.py's);
  * parity with HF fp32 (tests/golden/nomic_golden.npz: 12 layers up to 2048 tokens, 2 layers up to 8192) and with the fp64
    oracle; bitwise invariance across batches, buckets and launch paths; a bge-base embedder beside it unchanged; the router
    over HTTP.

Parity bars (rel-L2 per item, against HF fp32 and against the fp64 oracle): nomic_refs.BARS by (layers, pooling), each at
least twice the emulated fp16-operand floor (nomic_refs.emulate_forward) that tests/golden/make_nomic_golden.py records on the
golden cases; tests/test_nomic_bert.py asserts it."""
import numpy as np
import pytest

import os
from types import SimpleNamespace

import kernel_refs as KR
import nomic_refs as N
import test_gpu_forward_chain as FC
import test_gpu_full_wave_chain as FW
from oracle import bge_ref as R

gpu = pytest.mark.gpu

PARITY_BAR = 1e-3


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16 if np.asarray(a).dtype == np.float16 else np.uint32)


def _rel(a, b):
    return np.linalg.norm(np.asarray(a, np.float64) - b, axis=-1) / np.linalg.norm(b, axis=-1)


def _stats(rng, M):
    """(sum, M2) partials of random rows of mean ~0.3, sd ~1.5."""
    y = rng.standard_normal((M, 768)) * 1.5 + 0.3
    return KR.partials(y).astype(np.float32)


def _ids(rng, lens, S, vocab=30528):
    ids = np.zeros((len(lens), S), np.int32)
    for i, n in enumerate(lens):
        ids[i, :n] = rng.integers(1000, vocab, n)
    return ids


# ------------------------------------------------------------------------------------------------ kernels

@gpu
@pytest.mark.parametrize("M,S", [(1, 64), (100, 64), (129, 128), (300, 192), (512, 512)])
@pytest.mark.parametrize("ln", [True, False])
def test_gemm_rope(rt, M, S, ln):
    rng = np.random.default_rng(M + S)
    a = (rng.standard_normal((M, 768)) * 1.2).astype(np.float16)
    w = (rng.standard_normal((2304, 768)) * 0.05).astype(np.float16)
    c = (rng.standard_normal(2304) * 0.1).astype(np.float32)
    st = _stats(rng, M) if ln else None
    table = N.rope_table(S, 1000.0)
    out = rt.debug_gemm_rope(a, w, c, st, table, S, 1536, 1e-12)
    ref, tol = N.rope_gemm_ref(a, w, c, st, table, S, 1536, 1e-12)
    KR.check(f"gemm_rope M={M} S={S} ln={ln}", out.astype(np.float64), ref, tol)


@gpu
@pytest.mark.parametrize("M", [1, 100, 129, 300])
@pytest.mark.parametrize("ln", [True, False])
def test_gemm_swiglu(rt, M, ln):
    rng = np.random.default_rng(M)
    a = (rng.standard_normal((M, 768)) * 1.2).astype(np.float16)
    gate = rng.standard_normal((3072, 768)) * 0.05
    up = rng.standard_normal((3072, 768)) * 0.05
    w = N.interleave_rows(gate, up).astype(np.float16)
    c = N.interleave_rows(rng.standard_normal((3072, 1)), rng.standard_normal((3072, 1)))[:, 0].astype(np.float32) * 0.3
    st = _stats(rng, M) if ln else None
    out = rt.debug_gemm_swiglu(a, w, c, st, 1e-12)
    ref, tol = N.swiglu_gemm_ref(a, w, c, st, 1e-12)
    KR.check(f"gemm_swiglu M={M} ln={ln}", out.astype(np.float64), ref, tol)


def _attn_rows(S):
    """Query rows checked: all of them up to 1024, else a sample that covers every tile edge region."""
    if S <= 1024:
        return np.arange(S)
    r = np.unique(np.concatenate([np.arange(0, 130), np.arange(S // 2 - 70, S // 2 + 70), np.arange(S - 130, S),
                                  np.random.default_rng(S).integers(0, S, 64)]))
    return r


ATTN_CASES = [(64, [64, 1, 33]), (576, [576, 127, 128, 129, 1]), (1024, [1024, 1000, 513]), (2048, [2048, 129, 1500]),
              (4096, [4096, 2049]), (8192, [8191, 8192])]


@gpu
@pytest.mark.parametrize("S,lens", ATTN_CASES)
def test_attention_stream(rt, S, lens):
    B = len(lens)
    qkv = N.synth_qkv(B, S, S, q_scale=0.5)
    ctx, _ = rt.debug_attention_stream(qkv, np.array(lens, np.int32), B, S)
    rows = _attn_rows(S)
    ref, tol = N.attention_rows_ref(qkv, lens, B, S, rows)
    got = ctx.reshape(B, S, 768)[:, rows].astype(np.float64)
    assert np.isfinite(ctx.astype(np.float32)).all()
    KR.check(f"attention_stream S={S} lens={lens}", got, ref, tol)


@gpu
def test_attention_stream_zero_q(rt):
    """Q = 0: every score is 0, ctx is the plain mean of the valid V rows."""
    S, lens = 640, [600, 1]
    qkv = N.synth_qkv(2, S, 7)
    qkv[:, :768] = 0
    ctx, _ = rt.debug_attention_stream(qkv, np.array(lens, np.int32), 2, S)
    ref, tol = N.attention_rows_ref(qkv, lens, 2, S, np.arange(S))
    KR.check("attention_stream Q=0", ctx.reshape(2, S, 768).astype(np.float64), ref, tol)


@gpu
@pytest.mark.parametrize("S,lens", [(2048, [2048, 700, 5]), (8192, [8192])])
def test_attention_stream_grid_invariance(rt, S, lens):
    qkv = N.synth_qkv(len(lens), S, 11, q_scale=0.5)
    l = np.array(lens, np.int32)
    a, _ = rt.debug_attention_stream(qkv, l, len(lens), S, sms=1)
    b, _ = rt.debug_attention_stream(qkv, l, len(lens), S, sms=0)
    c, _ = rt.debug_attention_stream(qkv, l, len(lens), S, sms=7)
    assert (_bits(a) == _bits(b)).all() and (_bits(a) == _bits(c)).all()


# ---- the streaming kernel at every launch width the runtime uses
#
# A CTA walks units u = blockIdx.x, + gridDim.x, ... (grid = min(units, sms)); each unit pushes its item's ceil(len / 128)
# key tiles through a 4-stage K/V ring whose phase bit flips on every wrap, and the ring carries over from one unit to the
# next.  On one CTA every item starts at stage 0, because its 12 nq units are a multiple of 4: only odd tile counts, and
# widths other than 1, move the stage a unit starts at.  stream_walk restates that walk (attention_sm90.cu,
# attention_stream_kernel's producer loop), and test_stream_walk_covers_the_ring checks that the cases below start units at
# every stage on both phases, wrap the ring inside a unit and change the tile count between a CTA's consecutive units.

STREAM_NSTAGE = 4
H100_SMS = 132


def stream_walk(lens, S, sms):
    """Per CTA, the units it walks in order, as (unit, key tiles, ring stage and phase the unit starts at)."""
    nq = (S + 127) // 128
    n_units = len(lens) * 12 * nq
    grid = min(n_units, sms or H100_SMS)
    walks = []
    for cta in range(grid):
        stage, phase, walk = 0, 0, []
        for u in range(cta, n_units, grid):
            tiles = (min(max(int(lens[u // nq // 12]), 1), S) + 127) // 128
            walk.append((u, tiles, stage, phase))
            stage += tiles
            phase ^= (stage // STREAM_NSTAGE) & 1
            stage %= STREAM_NSTAGE
        walks.append(walk)
    return walks


# many units per CTA: 8 items of 1024 tokens, key tiles 1, 2, 3, 4, 5, 6, 8, 8
STREAM_MANY = (1024, [1, 129, 300, 385, 640, 700, 897, 1024])
STREAM_MANY_SMS = (1, 2, 3, 5, 12, 13, 21, 66, 111, 131)
# fewer units than CTAs: 12 and 24 units
STREAM_FEW = [(128, [128]), (256, [200])]
STREAM_FEW_SMS = (0, 13, 23, 25)


def _stream_cases():
    yield from ((STREAM_MANY[0], STREAM_MANY[1], sms) for sms in (0,) + STREAM_MANY_SMS)
    yield from ((S, lens, sms) for S, lens in STREAM_FEW for sms in STREAM_FEW_SMS)


def test_stream_walk_covers_the_ring():
    starts, wraps, changes = set(), False, False
    for S, lens, sms in _stream_cases():
        for walk in stream_walk(lens, S, sms):
            for i, (u, tiles, stage, phase) in enumerate(walk):
                starts.add((stage, phase))
                wraps |= tiles == 3 and stage >= 2
                changes |= i > 0 and walk[i - 1][1] != tiles
    assert starts == {(st, ph) for st in range(STREAM_NSTAGE) for ph in (0, 1)}, starts
    assert wraps and changes
    # on one CTA every item's first unit starts at stage 0
    walk = stream_walk(STREAM_MANY[1], STREAM_MANY[0], 1)[0]
    assert {stage for u, _, stage, _ in walk if u % (12 * 8) == 0} == {0}


@gpu
def test_attention_stream_many_units_per_cta(rt):
    """Every row of the 8 items on every SM against the fp64 reference; then bitwise the same at the widths of
    STREAM_MANY_SMS, 1 (all 768 units on one CTA) to 131, the split runtime's 21 and 66 among them."""
    S, lens = STREAM_MANY
    B = len(lens)
    qkv = N.synth_qkv(B, S, 17, q_scale=0.5)
    l = np.array(lens, np.int32)
    base, _ = rt.debug_attention_stream(qkv, l, B, S)
    ref, tol = N.attention_rows_ref(qkv, lens, B, S, np.arange(S))
    KR.check(f"attention_stream S={S} lens={lens} every SM", base.reshape(B, S, 768).astype(np.float64), ref, tol)
    for sms in STREAM_MANY_SMS:
        got, _ = rt.debug_attention_stream(qkv, l, B, S, sms=sms)
        same = (_bits(got) == _bits(base)).all()
        print(f"attention_stream S={S}: sms {sms} ({min(sms, B * 12 * 8)} CTAs) bitwise equal to every SM: {same}")
        assert same, sms


@gpu
@pytest.mark.parametrize("S,lens", STREAM_FEW)
def test_attention_stream_fewer_units_than_ctas(rt, S, lens):
    B = len(lens)
    qkv = N.synth_qkv(B, S, S + 3, q_scale=0.5)
    l = np.array(lens, np.int32)
    ref, tol = N.attention_rows_ref(qkv, lens, B, S, np.arange(S))
    first = None
    for sms in STREAM_FEW_SMS:
        got, _ = rt.debug_attention_stream(qkv, l, B, S, sms=sms)
        KR.check(f"attention_stream S={S} lens={lens} sms {sms}", got.reshape(B, S, 768).astype(np.float64), ref, tol)
        first = got if first is None else first
        assert (_bits(got) == _bits(first)).all(), sms


@gpu
@pytest.mark.parametrize("S", list(range(64, 513, 64)))
def test_attention_stream_matches_resident_kernel_bitwise(rt, S):
    """At S <= 512 the streaming kernel's ctx is attention_kernel<64, 12>'s, bit for bit, in both of the resident kernel's
    unit layouts (split by query tile for small batches, whole heads for large ones)."""
    rng = np.random.default_rng(S)
    for B in (2, 12):
        lens = rng.integers(1, S + 1, B).astype(np.int32)
        lens[0] = S
        qkv = N.synth_qkv(B, S, S + B, q_scale=0.7)
        a, _ = rt.debug_attention_stream(qkv, lens, B, S)
        b, _ = rt.debug_attention(qkv, lens, B, S)
        assert (_bits(a) == _bits(b)).all(), (S, B, int((_bits(a) != _bits(b)).sum()))


# ------------------------------------------------------------------------------------------------ model

def _model(rt, g, flat, pooling="mean"):
    return rt.NomicEmbedModel(g, N.pack(flat, g), pooling=pooling)


@gpu
def test_forward_launches(rt):
    g = N.geometry(layers=2, max_pos=1024)
    m = _model(rt, g, N.make_weights(g, 1, "hf"))
    rng = np.random.default_rng(0)
    ids = _ids(rng, [128, 77], 128)
    tr = m.debug_trace(ids, [128, 77], 12)
    assert tr["n_total"] == 12
    assert tr["names"] == ["embed"] + ["gemm_qkv_rope", "attention_stream", "gemm_attn_out", "gemm_ffn1_swiglu", "gemm_ffn2"] * 2 + \
        ["mean_pool_normalize"]
    assert (_bits(tr["out"]) == _bits(m.embed(ids, [128, 77]))).all()
    # the embedding: LN(word + type0) as hi + lo, bit for bit the sum the row kernel forms: (word + type0) + 0
    flat = N.make_weights(g, 1, "hf")
    tr0 = m.debug_trace(ids, [128, 77], 1)
    x = (flat["emb.word"][ids.reshape(-1)] + flat["emb.type"][0]) + np.float32(0)
    hi = x.astype(np.float16)
    assert (_bits(tr0["yhi"][:256]) == _bits(hi)).all()
    assert (_bits(tr0["ylo"][:256]) == _bits((x - hi.astype(np.float32)).astype(np.float16))).all()


class NomicChain(FC.TextChain):
    """TextChain of a nomic-bert model: the engine's weights rebuilt from the flat tensors (each projection's LayerNorm folded by
    the GPU fold, gate / up interleaved in groups of 8 here, so the engine's own interleave is checked too), and the checks of
    gemm_qkv_rope (the rotary reference at each row's position), attention_stream, the zero-bias residual epilogues and
    gemm_ffn1_swiglu.  run_chain counts layers by "gemm_qkv", so the chain counts them itself."""

    def __init__(self, flat, g, ids, lens, fold, rows=None):
        self.flat, self.ids, self.lens = flat, np.asarray(ids, np.int32), np.asarray(lens, np.int32)
        self.g = SimpleNamespace(hidden=768, heads=12, inter=3072, layers=g["layers"], eps=g["eps"], vocab=g["vocab"])
        self.B, self.S = self.ids.shape
        self.M = self.B * self.S
        self.hd = 64
        FC.set_rows(self, rows)
        self.pos = np.arange(self.M)[self.rows] % self.S
        self.table = N.rope_table(self.S, g["rope_theta"])
        f = flat
        self.qkv, self.ff1, self.ao16, self.ff216 = [], [], [], []
        for l in range(g["layers"]):
            p = f"l{l}."
            lg, lb = self.prev_ln(l)
            self.qkv.append(fold(f[p + "qkv.w"], lg, lb, None))
            self.ff1.append(fold(N.interleave_rows(f[p + "gate.w"], f[p + "up.w"]), f[p + "ln1.g"], f[p + "ln1.b"], None))
            self.ao16.append(fold(f[p + "ao.w"])[0])
            self.ff216.append(fold(f[p + "down.w"])[0])
        self.layer = -1

    def check(self, tag, name, l, prev, cur):
        M, f, eps = self.M, self.flat, self.g.eps
        P = lambda t, b: t[b][self.rows]  # noqa: E731
        A = lambda t, b: t[b][:M]  # noqa: E731
        if name == "embed":
            self.layer = -1
            return KR.check_embed(f"{tag} embed", A(cur, "yhi"), A(cur, "ylo"), P(cur, "pstats0"), self.ids.reshape(-1), f["emb.word"],
                                  np.zeros((64, 768), np.float32), f["emb.type"][0], 64, rows=self.rows)
        self.layer += name == "gemm_qkv_rope"
        l, p = self.layer, f"l{self.layer}."
        what = f"{tag} layer {l} {name}"
        zero = np.zeros(768, np.float32)
        if name == "gemm_qkv_rope":
            w16, c = self.qkv[l]
            ref, tol = N.rope_gemm_ref(P(prev, "yhi"), w16, c, P(prev, "pstats0"), self.table, self.S, 1536, eps, pos=self.pos)
            return KR.check(what, P(cur, "qkv").astype(np.float64), ref, tol)
        if name == "attention_stream":
            return KR.check_attention(what, P(cur, "ctx"), A(prev, "qkv"), self.lens, self.B, self.S, rows=self.q_rows)
        if name == "gemm_attn_out":
            kw = dict(resid_hilo=(P(prev, "yhi"), P(prev, "ylo")), ln_stats=P(prev, "pstats0"), ln_gamma=self.prev_ln(l)[0],
                      ln_beta=self.prev_ln(l)[1], eps=eps)
            return FC._check_residual(what, cur, "pstats1", self.rows, (P(prev, "ctx"), self.ao16[l], zero), kw)
        if name == "gemm_ffn1_swiglu":
            w16, c = self.ff1[l]
            ref, tol = N.swiglu_gemm_ref(P(prev, "yhi"), w16, c, P(prev, "pstats1"), eps)
            return KR.check(what, P(cur, "ffn").astype(np.float64), ref, tol)
        if name == "gemm_ffn2":
            kw = dict(resid_hilo=(P(prev, "yhi"), P(prev, "ylo")), ln_stats=P(prev, "pstats1"), ln_gamma=f[p + "ln1.g"],
                      ln_beta=f[p + "ln1.b"], eps=eps)
            return FC._check_residual(what, cur, "pstats0", self.rows, (P(prev, "ffn"), self.ff216[l], zero), kw)
        return super().check(tag, name, l, prev, cur)


@pytest.fixture
def nomic_launches(monkeypatch):
    """run_chain's table of the buffers each launch writes, extended by the kind's three launches."""
    monkeypatch.setitem(FC.WRITES, "gemm_qkv_rope", ("qkv",))
    monkeypatch.setitem(FC.WRITES, "attention_stream", ("ctx",))
    monkeypatch.setitem(FC.WRITES, "gemm_ffn1_swiglu", ("ffn",))


@gpu
@pytest.mark.parametrize("style,pooling,lens,S", [("trained", "mean", [704, 1, 129, 513], 704), ("hf", "cls", [192, 1, 64, 65, 130], 192)])
def test_forward_chain(rt, nomic_launches, style, pooling, lens, S):
    """2 layers on a toy ragged batch, every launch against its reference on the operands it consumed; the 704 bucket takes
    six key tiles, more than one lap of the four-stage ring."""
    g = N.geometry(layers=2, max_pos=1024)
    flat = N.make_weights(g, 8, style)
    m = _model(rt, g, flat, pooling)
    ids = _ids(np.random.default_rng(S), lens, S)
    ch = NomicChain(flat, g, ids, lens, FC.gpu_fold(rt))
    margins = {}
    last = FC.run_chain(f"nomic {style} {S}", ch, lambda k: m.debug_trace(ids, lens, k), margins, m.debug_cap_rows())
    FC.print_margins(f"nomic {style} {pooling} {lens} @ {S}", margins)
    assert last["n_total"] == 5 * 2 + 2
    assert (_bits(m.embed(ids, np.array(lens, np.int32))) == _bits(last["out"])).all()


def full_wave_rows(B, S):
    """tests/test_gpu_full_wave_chain.py's row sample of a B x S wave, except that the first and last items are read at their
    edges (192 rows each end) and every 61st row rather than whole (a whole 8192-token item would need [12, 8192, 8192] fp64
    attention scores), plus one row of every 64-row GEMM half tile."""
    rows = FW.sample_rows(B, S)
    item, w = rows // S, rows % S
    keep = ((item > 0) & (item < B - 1)) | (w < 192) | (w >= S - 192) | (w % 61 == 0)
    h = np.arange(B * S // 64)
    return np.unique(np.concatenate([rows[keep], h * 64 + (h * 37) % 64]))


@gpu
def test_full_wave_chain_8192(rt, nomic_launches):
    """One full wave of the 8192 bucket (8 items on an H100 SXM), 2 layers, every launch checked on the row sample."""
    g = N.geometry(layers=2, max_pos=8192)
    flat = N.make_weights(g, 9, "trained")
    m = _model(rt, g, flat)
    S = 8192
    B = m.debug_cap_rows() // S
    rng = np.random.default_rng(3)
    lens = rng.integers(7000, S + 1, B).astype(np.int32)
    lens[0] = S
    ids = _ids(rng, lens, S)
    ch = NomicChain(flat, g, ids, lens, FC.gpu_fold(rt), rows=full_wave_rows(B, S))
    margins = {}
    FC.run_chain(f"nomic full wave {B} x {S}", ch, lambda k: m.debug_trace(ids, lens, k), margins, m.debug_cap_rows())
    FC.print_margins(f"nomic full wave {B} x {S}", margins)


GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nomic_golden.npz"))
GOLDEN_CASES = ("l12_hf", "l12_trained", "l2_hf_8k", "l2_trained_8k")


@gpu
@pytest.mark.parametrize("case", GOLDEN_CASES)
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_parity_with_hf_golden(rt, case, pooling):
    """The engine against HF fp32 NomicBertModel (tests/golden/make_nomic_golden.py), at nomic_refs.BARS."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_nomic_golden", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                                                                    "make_nomic_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    layers, max_pos, style, seed, _ = mg.CASES[case]
    g = N.geometry(layers=layers, max_pos=max_pos)
    m = _model(rt, g, N.make_weights(g, seed, style), pooling)
    ids, lens = GOLDEN[f"{case}_ids"], GOLDEN[f"{case}_lens"]
    rel = _rel(m.embed(ids, lens), GOLDEN[f"{case}_{pooling}"].astype(np.float64))
    bar = N.BARS[(layers, pooling)]
    floor = GOLDEN[f"{case}_floor_{pooling}"].max()
    print(f"nomic {case} {pooling} vs HF fp32, lens {lens.tolist()}: rel-L2 {' '.join(f'{r:.2e}' for r in rel)} "
          f"(bar {bar}, emulated floor {floor:.2e})")
    assert rel.max() < bar, rel


_HIDDEN = {}


@gpu
@pytest.mark.parametrize("layers,style,lens,max_pos", [
    (2, "hf", [2048, 1500, 513, 64, 3], 2048),
    (2, "trained", [2048, 1000, 600, 129, 1], 2048),
    (12, "trained", [2048, 700, 100], 2048),
    (2, "trained", [8192, 4097, 1000, 513], 8192),
])
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_parity_with_fp64_oracle(rt, layers, style, lens, max_pos, pooling):
    g = N.geometry(layers=layers, max_pos=max_pos)
    flat = N.make_weights(g, 5, style)
    m = _model(rt, g, flat, pooling)
    rng = np.random.default_rng(layers + max_pos)
    ids = _ids(rng, lens, max(lens))
    got = m.embed(ids, np.array(lens, np.int32))
    key = (layers, style, tuple(lens), max_pos)
    if key not in _HIDDEN:  # the fp64 hidden states serve both poolings
        _HIDDEN[key] = N.hidden_np(flat, ids, lens, g)
    ref = N.pool(_HIDDEN[key], pooling)
    rel = _rel(got, ref)
    bar = N.BARS[(layers, pooling)]
    print(f"nomic {layers} layers {style} {pooling} lens {lens}: rel-L2 {' '.join(f'{r:.2e}' for r in rel)} (bar {bar})")
    assert rel.max() < bar, rel


@gpu
def test_full_wave_of_8192_token_items(rt):
    """One full wave of the 8192 bucket (8 items on an H100 SXM): every item within the bar of the oracle (checked on three of
    them: the fp64 oracle takes ~1 min per 8192-token item at 2 layers), and bitwise the item's embedding alone."""
    g = N.geometry(layers=2, max_pos=8192)
    flat = N.make_weights(g, 9, "trained")
    m = _model(rt, g, flat)
    B = m.debug_cap_rows() // 8192
    rng = np.random.default_rng(3)
    lens = rng.integers(7000, 8193, B).astype(np.int32)
    lens[0] = 8192
    ids = _ids(rng, lens, 8192)
    got = m.embed(ids, lens)
    assert np.isfinite(got).all()
    for i in (0, B // 2, B - 1):
        ref = N.forward_np(flat, ids[i:i + 1], lens[i:i + 1], g)
        rel = _rel(got[i:i + 1], ref)[0]
        print(f"full wave item {i} len {lens[i]}: rel-L2 {rel:.2e}")
        assert rel < PARITY_BAR
        assert (_bits(m.embed(ids[i:i + 1, :lens[i]], lens[i:i + 1])) == _bits(got[i:i + 1])).all()


@gpu
def test_bitwise_invariance_across_batches_buckets_and_paths(rt):
    import torch

    g = N.geometry(layers=2, max_pos=8192)
    m = _model(rt, g, N.make_weights(g, 2, "trained"))
    rng = np.random.default_rng(4)
    lens = np.array([1500, 64, 8000, 300, 2048, 1, 4097], np.int32)
    ids = _ids(rng, lens, 8192)
    mixed = m.embed(ids, lens)  # ragged: items span the 64 ... 8192 buckets and come back in order
    for i in range(len(lens)):
        alone = m.embed(ids[i:i + 1, :lens[i]], lens[i:i + 1])
        assert (_bits(alone) == _bits(mixed[i:i + 1])).all(), i
    # a 1500-token item through embed_device at max_len 2048 and 4096 (longer buckets than its own)
    with torch.cuda.device(0):
        for S in (2048, 4096):
            d_ids = torch.from_numpy(np.ascontiguousarray(ids[:1, :S])).cuda()
            d_lens = torch.from_numpy(lens[:1].copy()).cuda()
            d_out = torch.empty((1, 768), dtype=torch.float32, device="cuda")
            m.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), 1, S, d_out.data_ptr(), 0)
            rt.device_sync(0)
            assert (_bits(d_out.cpu().numpy()) == _bits(mixed[:1])).all(), S


@gpu
def test_bge_base_beside_nomic_is_unchanged(rt):
    bg = R.BertGeometry(layers=2)
    bflat = R.make_weights(bg, 3, "trained")
    ids, lens = R.synth_ragged(6, 300, seed=2, min_len=3)
    bge = rt.EmbedModel(R.geometry_dict(bg), R.pack_blob(bflat, bg), pooling="mean")
    before = bge.embed(ids, lens)
    g = N.geometry(layers=2, max_pos=8192)
    nm = _model(rt, g, N.make_weights(g, 2, "hf"))
    nm.embed(_ids(np.random.default_rng(1), [5000, 100], 5000), np.array([5000, 100], np.int32))
    after = bge.embed(ids, lens)
    assert (_bits(before) == _bits(after)).all()


@gpu
def test_load_refusals(rt):
    g = N.geometry(layers=1, max_pos=8192)
    blob = N.pack(N.make_weights(g, 0, "hf"), g)
    for bad in (dict(max_pos=8193), dict(hidden=384), dict(inter=4096), dict(rope_theta=0.0)):
        gg = dict(g, **bad)
        with pytest.raises(rt.B200RTError) as e:
            rt.NomicEmbedModel(gg, blob)
        assert e.value.code == rt.E_UNSUPPORTED
    m = rt.NomicEmbedModel(g, blob)
    with pytest.raises(rt.B200RTError):  # segments are a classifier's
        m._submit(np.ones((1, 64), np.int32), None, np.zeros(1, np.int32), None, None, False)
    with pytest.raises(rt.B200RTError):  # past max_pos
        m.embed(np.ones((1, 8193), np.int32))


@gpu
def test_router_embeds_a_long_input_on_seeded_weights(rt):
    """text-embeddings-router --model-id nomic-ai/nomic-embed-text-v1.5 offline, over HTTP: seeded weights of the 12-layer
    geometry, GET /info reports the long max_input_length, and POST /embed of a ~3000-token input answers within the bar of the
    fp64 oracle on the same ids; past 8192 tokens it answers 413, or embeds the first 8192 with "truncate": true."""
    from b200rt import weights as W
    from tei_router import server

    import test_nomic_bert as TN

    rt.shutdown()  # the router's engine initialises the runtime itself
    try:
        e = server.Engine(server.parse_args(["--model-id", "nomic-ai/nomic-embed-text-v1.5", "--gpus", "1"]))
        e.args.auto_truncate = False  # the synthetic vocabulary turns it on; TEI's request-level truncate is what is tested
        post, get, stop = TN.serve(e)
        try:
            code, info = get("/info")
            assert code == 200 and info["max_input_length"] == 8192 and info["pooling"] == "mean"
            text = " ".join(f"word{i % 97} token" for i in range(600))
            ids = np.array([e.tok.encode(text, 8192)], np.int32)
            assert 1500 <= ids.shape[1] <= 8192, ids.shape
            code, body = post("/embed", {"inputs": text})
            assert code == 200
            g = W.NOMIC_EMBED_TEXT_GEOMETRY
            flat = N.unpack(W.random_nomic_blob(g, 0), g)
            rel = _rel(np.array(body, np.float64), N.forward_np(flat, ids, [ids.shape[1]], g))[0]
            print(f"router POST /embed of {ids.shape[1]} tokens vs fp64 oracle: rel-L2 {rel:.2e}")
            assert rel < N.BARS[(12, "mean")]
            long_text = " ".join(f"word{i % 97} token" for i in range(3000))
            assert post("/embed", {"inputs": long_text})[0] == 413
            code, body = post("/embed", {"inputs": long_text, "truncate": True})
            assert code == 200 and np.isfinite(np.array(body)).all()
        finally:
            stop()
    finally:
        rt.shutdown()
        rt.init(devices=[0])
