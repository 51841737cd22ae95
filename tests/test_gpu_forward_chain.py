"""Forward-chain conformance: every launch of the product forward, checked at kernel precision on the operands it consumed.

`EmbedModel.debug_trace(ids, lens, k)` / `ImageEmbedModel.debug_trace(pixels, k)` poison the workspace (0xFF bytes: NaN in
fp16 and fp32), run the first k launches of the forward exactly as the product enqueues them, and return every workspace
buffer for M + 256 rows.  Traces k - 1 and k are then the inputs and the output of launch k, which is checked against the
fp64 reference of its kernel (tests/kernel_refs.py, tests/attention_refs.py) at that reference's tolerance, with the weights
the engine folded at load time (the QKV of layer l folds the embedding LayerNorm at l = 0 and LN2 of layer l - 1 after that;
FFN1 folds LN1).  What that adds to the kernel tests is the wiring between launches: which buffer each launch reads and
writes, which statistics buffer, which LayerNorm a residual epilogue re-applies and which hi / lo pair it updates in place.
At every launch:
  * every buffer the launch does not write is bitwise what the previous launch left, and a written buffer is unchanged past
    the rows the launch owns;
  * rows >= M of every buffer are still poison;
  * every row < M the launch wrote is finite, padded tokens included.
A model-level comparison (rel-L2 1e-3 against the oracle) cannot see a lost `lo` half of the residual stream; these checks
can, and the CPU tests at the end show it: a numpy emulation of a 2-layer chain passes them, and each wiring mutant fails.

The GPU tests carry `@gpu`."""
import hashlib
import time

import numpy as np
import pytest

import attention_refs as AR
import kernel_emul as KE
import kernel_refs as KR
import mean_pool_refs as MP
from oracle import bge_ref as R
from oracle import clip_ref as C

gpu = pytest.mark.gpu

BUFFERS = ("yhi", "ylo", "pstats0", "pstats1", "qkv", "ctx", "ffn")
GUARD = 256  # rows past M a trace returns, as far as the model's capacity allows
# the workspace buffers each launch writes (the pool launches write only `out`)
WRITES = {
    "embed": ("yhi", "ylo", "pstats0"), "gemm_qkv": ("qkv",), "attention": ("ctx",), "gemm_attn_out": ("yhi", "ylo", "pstats1"),
    "gemm_ffn1_gelu": ("ffn",), "gemm_ffn2": ("yhi", "ylo", "pstats0"), "pool_normalize": (),
    "im2col": ("ffn",), "gemm_patch": ("ctx",), "vit_embed": ("yhi", "ylo", "pstats0"), "gemm_ffn1_qgelu": ("ffn",), "vit_pool": (),
    "mean_pool_normalize": (), "clip_text_pool": (),
}
POOLS = ("pool_normalize", "vit_pool", "mean_pool_normalize", "clip_text_pool")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.reshape(-1).view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _poison_bits(a):
    return 0xFFFF if a.dtype == np.float16 else 0xFFFFFFFF


def _im2col_cols(ch):
    return 3 * ch.g.patch * ch.g.patch


def check_invariants(tag, name, prev, cur, ch):
    """The buffer-level invariants of launch `name` (trace prev -> cur)."""
    M = ch.M
    for buf in BUFFERS:
        p, c = _bits(prev[buf]), _bits(cur[buf])
        row = p.size // prev[buf].shape[0]
        written = M * (_im2col_cols(ch) if name == "im2col" else row)  # im2col: [M, 3 p p] at the start of ffn
        if buf in WRITES[name]:
            assert np.array_equal(p[written:], c[written:]), f"{tag}: {name} wrote {buf} past its {M} rows"
            vals = np.asarray(cur[buf]).reshape(-1)[:written]
            assert np.isfinite(vals).all(), f"{tag}: {name} left {int((~np.isfinite(vals)).sum())} non-finite values in {buf} rows < M"
        else:
            assert np.array_equal(p, c), f"{tag}: {name} changed {buf}, which it does not own ({int((p != c).sum())} values)"
        assert (c[M * row:] == _poison_bits(cur[buf])).all(), f"{tag}: {name}: guard rows >= {M} of {buf} are not poison"
    if name in POOLS:
        assert np.isfinite(cur["out"]).all(), f"{tag}: {name}: non-finite pooled output"


def set_rows(ch, rows):
    """The rows the row-wise checks of `ch` read: all M (rows None) or an ascending sample.  Sets ch.rows (an index into the
    first M rows) and ch.q_rows (None, or each item's sampled rows within the item, for the attention references)."""
    if rows is None:
        ch.rows, ch.q_rows = slice(0, ch.M), None
        return
    rows = np.asarray(rows, np.int64)
    assert (np.diff(rows) > 0).all() and rows[0] >= 0 and rows[-1] < ch.M, "rows must be ascending and below M"
    ch.rows = rows
    cut = np.searchsorted(rows, np.arange(ch.B + 1) * ch.S)
    ch.q_rows = [rows[cut[b]:cut[b + 1]] - b * ch.S for b in range(ch.B)]


class TextChain:
    """A text encoder's weights as the engine holds them, the batch, and the check of each launch.  `fold(w, gamma, beta, bias)`
    gives the fp16 folded weight and cvec (gamma None: fp16(w), None).  `rows` (ascending, < M): check the GEMM, attention and
    statistics outputs on those rows only, every column of each; the embedding's bits and the pools are checked in full."""

    def __init__(self, flat, g, ids, lens, fold, rows=None):
        self.flat, self.g, self.ids, self.lens = flat, g, np.asarray(ids, np.int32), np.asarray(lens, np.int32)
        self.B, self.S = self.ids.shape
        self.M = self.B * self.S
        self.hd = g.hidden // g.heads
        set_rows(self, rows)
        f = flat
        self.qkv, self.ff1, self.ao16, self.ff216 = [], [], [], []
        for l in range(g.layers):
            p = f"l{l}."
            prev_ln = ("emb.ln.g", "emb.ln.b") if l == 0 else (f"l{l - 1}.ln2.g", f"l{l - 1}.ln2.b")
            self.qkv.append(fold(f[p + "qkv.w"], f[prev_ln[0]], f[prev_ln[1]], f[p + "qkv.b"]))
            self.ff1.append(fold(f[p + "ff1.w"], f[p + "ln1.g"], f[p + "ln1.b"], f[p + "ff1.b"]))
            self.ao16.append(fold(f[p + "ao.w"])[0])
            self.ff216.append(fold(f[p + "ff2.w"])[0])

    def prev_ln(self, l):
        """The LayerNorm that applies to the residual rows entering layer l."""
        f = self.flat
        return (f["emb.ln.g"], f["emb.ln.b"]) if l == 0 else (f[f"l{l - 1}.ln2.g"], f[f"l{l - 1}.ln2.b"])

    def check(self, tag, name, l, prev, cur):
        M, g, f, p = self.M, self.g, self.flat, f"l{l}."
        eps = g.eps
        P = lambda t, b: t[b][self.rows]  # noqa: E731
        A = lambda t, b: t[b][:M]  # noqa: E731
        what = f"{tag} layer {l} {name}"
        if name == "embed":
            return KR.check_embed(what, A(cur, "yhi"), A(cur, "ylo"), P(cur, "pstats0"), self.ids.reshape(-1), f["emb.word"],
                                  f["emb.pos"], f["emb.type"][0], self.S, rows=self.rows)
        if name == "gemm_qkv":
            w16, c = self.qkv[l]
            return KR.check_gemm(what, P(cur, "qkv"), 0, P(prev, "yhi"), w16, c, ln_stats=P(prev, "pstats0"), eps=eps)
        if name == "attention":
            if self.hd == 64 and g.heads == 12:
                return KR.check_attention(what, P(cur, "ctx"), A(prev, "qkv"), self.lens, self.B, self.S, rows=self.q_rows)
            return AR.check_attention(what, P(cur, "ctx"), A(prev, "qkv"), self.lens, self.B, self.S, heads=g.heads, head_dim=self.hd,
                                      rows=self.q_rows)
        if name in ("gemm_attn_out", "gemm_ffn2"):
            if name == "gemm_attn_out":
                a, w16, bias, (lg, lb), st_in, st_out = P(prev, "ctx"), self.ao16[l], f[p + "ao.b"], self.prev_ln(l), "pstats0", "pstats1"
            else:
                a, w16, bias, (lg, lb), st_in, st_out = P(prev, "ffn"), self.ff216[l], f[p + "ff2.b"], (f[p + "ln1.g"], f[p + "ln1.b"]), "pstats1", "pstats0"
            kw = dict(resid_hilo=(P(prev, "yhi"), P(prev, "ylo")), ln_stats=P(prev, st_in), ln_gamma=lg, ln_beta=lb, eps=eps)
            return _check_residual(what, cur, st_out, self.rows, (a, w16, bias), kw)
        if name == "gemm_ffn1_gelu":
            w16, c = self.ff1[l]
            return KR.check_gemm(what, P(cur, "ffn"), 1, P(prev, "yhi"), w16, c, ln_stats=P(prev, "pstats1"), eps=eps)
        if name == "pool_normalize":
            last = f"l{g.layers - 1}.ln2."
            return KR.check_pool_normalize(what, cur["out"], A(prev, "yhi"), A(prev, "ylo"), f[last + "g"], f[last + "b"], self.S, eps)
        if name == "mean_pool_normalize":
            last = f"l{g.layers - 1}.ln2."
            return MP.check_mean_pool_normalize(what, cur["out"], A(prev, "yhi"), A(prev, "ylo"), f[last + "g"], f[last + "b"], self.lens,
                                                self.S, eps)
        raise AssertionError(f"{tag}: unexpected launch {name!r}")


def _check_residual(what, cur, st_out, rows, args, kw):
    """A residual epilogue: the new hi + lo in place against the fp64 reference, hi the nearest fp16, and the partials of the new
    rows in `st_out` -- on `rows` (the operands in args / kw are those rows')."""
    hi, lo = cur["yhi"][rows], cur["ylo"][rows]
    m = KR.check_gemm(what, KR.hilo64(hi, lo), 2, *args, **kw)
    KR.hi_is_nearest(what, hi, lo)
    return max(m, KR.check_gemm_stats(f"{what} {st_out}", cur[st_out][rows], args, **kw))


def im2col_ref(pixels, g):
    """[n T, 3 p p] fp16: a zero row for the class token, then every patch flattened (channel, row, column), rounded to nearest."""
    n, p, gr = pixels.shape[0], g.patch, g.grid
    patches = pixels.reshape(n, 3, gr, p, gr, p).transpose(0, 2, 4, 1, 3, 5).reshape(n, gr * gr, 3 * p * p)
    return np.concatenate([np.zeros((n, 1, 3 * p * p), np.float32), patches], 1).reshape(n * g.tokens, -1).astype(np.float16)


class VitChain:
    """The ViT tower's weights as the engine holds them (LN1 folded into QKV, LN2 into FFN1, no LayerNorm re-applied to the
    residual), the batch, and the check of each launch.  `rows` as TextChain's (im2col, vit_embed and the pool in full)."""

    def __init__(self, flat, g, pixels, fold, rows=None):
        self.flat, self.g, self.pixels = flat, g, np.asarray(pixels, np.float32)
        self.B, self.S = self.pixels.shape[0], g.tokens
        self.M = self.B * self.S
        set_rows(self, rows)
        f = flat
        self.patch16 = fold(f["patch.w"])[0]
        self.qkv = [fold(f[f"l{l}.qkv.w"], f[f"l{l}.ln1.g"], f[f"l{l}.ln1.b"], f[f"l{l}.qkv.b"]) for l in range(g.layers)]
        self.ff1 = [fold(f[f"l{l}.ff1.w"], f[f"l{l}.ln2.g"], f[f"l{l}.ln2.b"], f[f"l{l}.ff1.b"]) for l in range(g.layers)]
        self.ao16 = [fold(f[f"l{l}.ao.w"])[0] for l in range(g.layers)]
        self.ff216 = [fold(f[f"l{l}.ff2.w"])[0] for l in range(g.layers)]

    def check(self, tag, name, l, prev, cur):
        M, g, f, p = self.M, self.g, self.flat, f"l{l}."
        eps, T = g.eps, self.S
        P = lambda t, b: t[b][self.rows]  # noqa: E731
        A = lambda t, b: t[b][:M]  # noqa: E731
        what = f"{tag} layer {l} {name}"
        im2col = lambda t: t["ffn"].reshape(-1)[:M * 3 * g.patch ** 2].reshape(M, -1)  # noqa: E731
        if name == "im2col":
            KR.check_bits(what, im2col(cur), im2col_ref(self.pixels, g))
            return 0.0
        if name == "gemm_patch":
            return KR.check_gemm(what, P(cur, "ctx"), 0, im2col(prev)[self.rows], self.patch16, np.zeros(g.hidden, np.float32))
        if name == "vit_embed":
            return KR.check_vit_embed(what, A(cur, "yhi"), A(cur, "ylo"), A(cur, "pstats0"), A(prev, "ctx"), f["cls"], f["pos"],
                                      f["pre.g"], f["pre.b"], T, eps)
        if name == "gemm_qkv":
            w16, c = self.qkv[l]
            return KR.check_gemm(what, P(cur, "qkv"), 0, P(prev, "yhi"), w16, c, ln_stats=P(prev, "pstats0"), eps=eps)
        if name == "attention":
            return KR.check_attention(what, P(cur, "ctx"), A(prev, "qkv"), [T] * self.B, self.B, T, rows=self.q_rows)
        if name == "gemm_attn_out":
            return _check_residual(what, cur, "pstats1", self.rows, (P(prev, "ctx"), self.ao16[l], f[p + "ao.b"]),
                                   dict(resid_hilo=(P(prev, "yhi"), P(prev, "ylo"))))
        if name == "gemm_ffn1_qgelu":
            w16, c = self.ff1[l]
            return KR.check_gemm(what, P(cur, "ffn"), 3, P(prev, "yhi"), w16, c, ln_stats=P(prev, "pstats1"), eps=eps)
        if name == "gemm_ffn2":
            return _check_residual(what, cur, "pstats0", self.rows, (P(prev, "ffn"), self.ff216[l], f[p + "ff2.b"]),
                                   dict(resid_hilo=(P(prev, "yhi"), P(prev, "ylo"))))
        if name == "vit_pool":
            return KR.check_vit_pool(what, cur["out"], A(prev, "yhi"), A(prev, "ylo"), f["post.g"], f["post.b"], f["proj.w"], T, eps)
        raise AssertionError(f"{tag}: unexpected launch {name!r}")


def run_chain(tag, ch, trace, margins=None, cap_rows=None):
    """Checks every launch of the forward: trace(k) is the workspace after k launches.  Holds two traces at a time; returns the
    last one and fills `margins` with the worst err / tol per launch name.  `cap_rows`: the model's workspace rows, which bound
    the rows a trace returns (at capacity there are no guard rows)."""
    margins = {} if margins is None else margins
    prev = trace(0)
    n_total = prev["n_total"]
    assert prev["names"] == [] and prev["rows"] == min(ch.M + GUARD, cap_rows or ch.M + GUARD)
    for buf in BUFFERS:
        assert (_bits(prev[buf]) == _poison_bits(prev[buf])).all(), f"{tag}: {buf} not poisoned before the first launch"
    layer = -1
    for k in range(1, n_total + 1):
        cur = trace(k)
        assert cur["names"][:-1] == prev["names"], (tag, k, cur["names"])
        name = cur["names"][-1]
        layer += name == "gemm_qkv"
        check_invariants(f"{tag} launch {k}", name, prev, cur, ch)
        m = ch.check(f"{tag} launch {k}", name, max(layer, 0), prev, cur)
        margins[name] = max(margins.get(name, 0.0), m)
        prev = cur
    assert prev["names"][-1] in POOLS
    return prev


def print_margins(tag, margins):
    print(f"\n{tag}: worst err/tol per launch")
    for name, m in margins.items():
        print(f"  {name:16s} {m:.3f}")


# ================================================================================================ GPU

_T0 = time.perf_counter()


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()
    print(f"\ntest_gpu_forward_chain: {time.perf_counter() - _T0:.1f} s wall time")


def gpu_fold(rt):
    return lambda w, gamma=None, beta=None, bias=None: rt.debug_fold_ln(w, gamma, beta, bias)


def ragged_batch(lens, S, seed):
    """ids [len(lens), S]: [CLS] ... [SEP] within each length, 0 ([PAD]) after it."""
    rng = np.random.default_rng(seed)
    ids = np.zeros((len(lens), S), np.int32)
    for i, n in enumerate(lens):
        ids[i, :n] = rng.integers(1000, 30522, size=n)
        ids[i, 0] = 101
        if n > 1:
            ids[i, n - 1] = 102
    return ids, np.asarray(lens, np.int32)


LENS5, S5 = [192, 1, 64, 65, 130], 192
GEOMETRIES = {"base": dict(), "small": dict(hidden=384, heads=12, inter=1536)}


def _text_case(rt, geometry, layers, style, seed):
    g = R.BertGeometry(layers=layers, **GEOMETRIES[geometry])
    flat = R.make_weights(g, seed, style)
    return g, flat, rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g))


def _trace_digest(t):
    return {b: hashlib.sha256(np.ascontiguousarray(t[b]).tobytes()).hexdigest() for b in BUFFERS + ("out",) if t[b] is not None}


@gpu
@pytest.mark.parametrize("geometry,style", [("base", "trained"), ("base", "hard"), ("small", "trained")])
def test_text_chain(rt, geometry, style):
    """2 layers, B = 5 ragged items padded to 192 (one item of a single token, lens on both sides of a 64-key sub-block).
    Then the product path: model.embed() of the same batch (scheduler, length buckets, CUDA-graph replay) is bitwise the
    traced pooled output, before and after another trace, and one forward is exactly 5 L + 2 launches (+ 1 scatter)."""
    g, flat, model = _text_case(rt, geometry, 2, style, 3)
    ids, lens = ragged_batch(LENS5, S5, seed=17)
    before = model.embed(ids, lens)
    ch = TextChain(flat, g, ids, lens, gpu_fold(rt))
    margins = {}
    last = run_chain(f"{geometry}/{style}", ch, lambda k: model.debug_trace(ids, lens, k), margins)
    print_margins(f"{geometry}/{style}", margins)
    assert last["n_total"] == 5 * g.layers + 2
    after = model.embed(ids, lens)
    for what, e in (("embed() before the traces", before), ("embed() after the traces", after)):
        same = np.array_equal(e.view(np.uint32), last["out"].view(np.uint32))
        print(f"{what}: bitwise the traced pooled output: {same}")
        assert same, what
    n0 = rt.stats()["kernel_launches"]
    model.embed(ids[:1], lens[:1])  # one item, one bucket: one wave
    n1 = rt.stats()["kernel_launches"]
    print(f"kernel launches of one {g.layers}-layer forward (+ the wave's scatter): {n1 - n0}")
    assert n1 - n0 == last["n_total"] + 1


@gpu
def test_vit_chain(rt):
    g = C.VitGeometry(layers=2)
    flat = C.make_weights(g, 1, "trained")
    model = rt.ImageEmbedModel(C.geometry_dict(g), C.pack_blob(flat, g))
    px = C.synth_pixels(3, g, 4)
    ch = VitChain(flat, g, px, gpu_fold(rt))
    margins = {}
    last = run_chain("vit", ch, lambda k: model.debug_trace(px, k), margins)
    print_margins("vit", margins)
    assert last["n_total"] == 5 * g.layers + 4
    e = model.embed(px)
    assert np.array_equal(e.view(np.uint32), last["out"].view(np.uint32)), "embed() differs from the traced pooled output"
    n0 = rt.stats()["kernel_launches"]
    model.embed(px)
    assert rt.stats()["kernel_launches"] - n0 == last["n_total"] + 1


@gpu
def test_text_chain_12_layers(rt):
    """bge-base, 12 layers, `hf` weights, B = 4 at S = 512: all 62 launches."""
    g, flat, model = _text_case(rt, "base", 12, "hf", 0)
    ids, lens = ragged_batch([512, 77, 300, 129], 512, seed=23)
    ch = TextChain(flat, g, ids, lens, gpu_fold(rt))
    margins = {}
    last = run_chain("base 12 layers", ch, lambda k: model.debug_trace(ids, lens, k), margins)
    print_margins("base 12 layers", margins)
    assert last["n_total"] == 62
    e = model.embed(ids, lens)
    assert np.array_equal(e.view(np.uint32), last["out"].view(np.uint32)), "embed() differs from the traced pooled output"


@gpu
def test_split_sm_traces_match_whole_gpu(rt):
    """B200RT_INIT_SPLIT_SMS(21): replica 0's GEMMs on 111 SMs, attention on 21.  Every trace of the bge-base 2-layer case is
    bitwise the whole-GPU runtime's.  The module's runtime is restarted around it."""
    ids, lens = ragged_batch(LENS5, S5, seed=17)

    def digests(flags):
        rt.shutdown()
        rt.init(devices=[0], flags=flags)
        _, _, model = _text_case(rt, "base", 2, "trained", 3)
        n = 5 * 2 + 2
        return [_trace_digest(model.debug_trace(ids, lens, k)) for k in range(n + 1)], rt.num_gpus()

    try:
        whole, n_whole = digests(0)
        split, n_split = digests(rt.SPLIT_SMS(21))
    finally:
        rt.shutdown()
        rt.init(devices=[0])
    assert n_whole == 1 and n_split == 2
    for k, (a, b) in enumerate(zip(whole, split)):
        assert a == b, f"launch {k}: {[n for n in a if a[n] != b.get(n)]} differ from the whole-GPU trace"
    print(f"split SMs k=21: all {len(whole)} traces bitwise equal to the whole-GPU runtime's")


# ================================================================================================ CPU: the chain checks discriminate

MUTANTS = ("stale_lo", "pool_zero_lo", "ffn1_pstats0", "attn_out_ln1", "guard_row", "foreign_buffer")


def emulate_chain(ch, mutant=None):
    """The traces of a text forward, emulated in numpy with the kernels' rounding (kernel_emul), as `debug_trace` returns them;
    `mutant` stands for a wiring bug:
      stale_lo        the residual epilogues update hi and leave lo as it was
      pool_zero_lo    the pool reads a zeroed lo
      ffn1_pstats0    FFN1 folds its LayerNorm with pstats0 (LN2's / the embedding's statistics) instead of pstats1
      attn_out_ln1    attention-out re-applies the layer's own LN1 instead of the LayerNorm in front of the layer
      guard_row       the QKV GEMM stores one row past M
      foreign_buffer  attention also writes a row of ffn"""
    g, f, M, S = ch.g, ch.flat, ch.M, ch.S
    H, I, P = g.hidden, g.inter, g.hidden // 128
    rows = M + GUARD
    f16 = lambda w: np.full((rows, w), 0xFFFF, np.uint16).view(np.float16)  # noqa: E731
    st = dict(yhi=f16(H), ylo=f16(H), qkv=f16(3 * H), ctx=f16(H), ffn=f16(I),
              pstats0=np.full((rows, P, 2), 0xFFFFFFFF, np.uint32).view(np.float32),
              pstats1=np.full((rows, P, 2), 0xFFFFFFFF, np.uint32).view(np.float32))
    n_total = 5 * g.layers + 2
    names = []
    traces = []

    def snap(name=None, out=None):
        if name:
            names.append(name)
        traces.append({**{k: v.copy() for k, v in st.items()}, "out": out, "names": list(names), "n_total": n_total, "M": M, "rows": rows})

    def residual(a, w16, bias, lg, lb, st_in, st_out):
        h, l, v = KE.emulate_gemm(2, a, w16, bias, resid_hilo=(st["yhi"][:M], st["ylo"][:M]), ln_stats=st[st_in][:M], ln_gamma=lg,
                                  ln_beta=lb, eps=g.eps, split=True)
        st["yhi"][:M] = h
        if mutant != "stale_lo":
            st["ylo"][:M] = l
        st[st_out][:M] = KE.partials32(v)

    snap()
    hi, lo, x = KR.embed_exact(ch.ids.reshape(-1), f["emb.word"], f["emb.pos"], f["emb.type"][0], S)
    st["yhi"][:M], st["ylo"][:M], st["pstats0"][:M] = hi, lo, KE.partials32(x)
    snap("embed")
    for l in range(g.layers):
        p = f"l{l}."
        w16, c = ch.qkv[l]
        st["qkv"][:M] = KE.emulate_gemm(0, st["yhi"][:M], w16, c, ln_stats=st["pstats0"][:M], eps=g.eps)
        if mutant == "guard_row":
            st["qkv"][M] = st["qkv"][M - 1]
        snap("gemm_qkv")
        st["ctx"][:M] = KE.emulate_attention(st["qkv"][:M], ch.lens, ch.B, S, head_dim=ch.hd)
        if mutant == "foreign_buffer":
            st["ffn"][0, :H] = st["ctx"][0]
        snap("attention")
        lg, lb = (f[p + "ln1.g"], f[p + "ln1.b"]) if mutant == "attn_out_ln1" else ch.prev_ln(l)
        residual(st["ctx"][:M], ch.ao16[l], f[p + "ao.b"], lg, lb, "pstats0", "pstats1")
        snap("gemm_attn_out")
        w16, c = ch.ff1[l]
        st["ffn"][:M] = KE.emulate_gemm(1, st["yhi"][:M], w16, c, ln_stats=st["pstats0" if mutant == "ffn1_pstats0" else "pstats1"][:M],
                                        eps=g.eps)
        snap("gemm_ffn1_gelu")
        residual(st["ffn"][:M], ch.ff216[l], f[p + "ff2.b"], f[p + "ln1.g"], f[p + "ln1.b"], "pstats1", "pstats0")
        snap("gemm_ffn2")
    last = f"l{g.layers - 1}.ln2."
    lo_rows = np.zeros_like(st["ylo"][:M:S]) if mutant == "pool_zero_lo" else st["ylo"][:M:S]
    x = st["yhi"][:M:S].astype(np.float32) + lo_rows.astype(np.float32)
    snap("pool_normalize", KE.l2_normalise32(KE.ln32(x, f[last + "g"], f[last + "b"], g.eps)))
    return traces


@pytest.fixture(scope="module")
def cpu_chain():
    """bge-base geometry, 2 layers, `trained` weights; B = 2 at S = 128, one item ragged."""
    g = R.BertGeometry(layers=2)
    flat = R.make_weights(g, 3, "trained")
    ids, lens = ragged_batch([128, 77], 128, seed=5)
    return TextChain(flat, g, ids, lens, KE.fold_ln32)


def test_chain_checks_accept_the_emulated_forward(cpu_chain):
    traces = emulate_chain(cpu_chain)
    margins = {}
    last = run_chain("emulated", cpu_chain, traces.__getitem__, margins)
    print_margins("emulated", margins)
    rel = R.rel_l2(last["out"], R.forward_np(cpu_chain.flat, cpu_chain.ids, cpu_chain.lens, cpu_chain.g))
    print(f"emulated forward: rel-L2 against the fp64 oracle {rel.max():.3e}")
    assert rel.max() < 1e-3


@pytest.mark.parametrize("mutant", MUTANTS)
def test_chain_checks_reject_wiring_mutants(cpu_chain, mutant):
    traces = emulate_chain(cpu_chain, mutant)
    if mutant in ("stale_lo", "pool_zero_lo"):  # invisible at the model level: within the 1e-3 bar of every parity test
        rel = R.rel_l2(traces[-1]["out"], R.forward_np(cpu_chain.flat, cpu_chain.ids, cpu_chain.lens, cpu_chain.g))
        print(f"mutant {mutant}: emulated end-to-end rel-L2 against the fp64 oracle {rel.max():.3e} (bar 1e-3)")
        assert rel.max() < 1e-3
    with pytest.raises(AssertionError) as e:
        run_chain(f"mutant {mutant}", cpu_chain, traces.__getitem__)
    print(f"mutant {mutant}: caught: {str(e.value).splitlines()[0][:160]}")
