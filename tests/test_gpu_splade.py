"""GPU: SPLADE sparse encoders (kind "bert_splade") -- the three launches the SPLADE head adds, the head launch by launch in
the real forward, parity with the fp64 oracle, bitwise invariance of an item's vector, and the router's /embed_sparse.

  * kernels: gemm_kernel<EPI_SPLADE_MAX> at K = 384 / 768 / 1024 and S = 64 / 512 with ragged lengths, the vocabulary's last
    column tile and lengths past S (clamped), against its fp64 reference, and bitwise the same on 1, 7 and every SM;
    mlm_ln_stats against the fp64 partials (and its zeroing of the max buffer); splade_finalize against log1p;
  * forward chain: 2-layer models on ragged batches through run_chain (tests/test_gpu_forward_chain.py) with a TextChain
    subclass that checks gemm_mlm_transform, mlm_ln_stats, gemm_splade and splade_finalize on the operands they consumed;
    embed(), the device-resident entry and the trace agree bitwise; then one full wave of the 128-token bucket on the row
    sample of tests/test_gpu_full_wave_chain.py;
  * parity: per-item rel-L2 and max |err| against the fp64 oracle and against HF fp32 (tests/golden/splade_golden.npz), the
    support wherever the reference is more than twice the bar away from 0, and the top words;
  * invariance: an item's vector is bitwise the same alone, inside a full wave of the 64- and 512-token buckets and at
    another padded length; an embedder and a reranker loaded beside it are bitwise unchanged."""
import importlib.util
import json
import os
import socket
import subprocess
import time
import urllib.request

import numpy as np
import pytest

import kernel_refs as KR
import rerank_refs as RR
import splade_refs as SR
import test_gpu_forward_chain as FC
import test_gpu_full_wave_chain as FW
from oracle import bge_ref as R

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "modal-examples_b200")
GOLDEN = os.path.join(ROOT, "tests", "golden")
_spec = importlib.util.spec_from_file_location("make_splade_golden", os.path.join(GOLDEN, "make_splade_golden.py"))
msg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(msg)
GEOMS = {"base": dict(), "small": dict(hidden=384, heads=12, inter=1536), "large": dict(hidden=1024, heads=16, inter=4096)}

# Parity bars against the fp64 oracle, per item: rel-L2 of the vocab-wide vector and max |err| over the vocabulary.  Their
# floor is what the fp16 GEMM operands of the head alone cost (splade_refs.splade_fp16_operands against the oracle, printed
# by test_parity_with_oracle beside the measured error).  On the 2-layer parity batch the floor is rel-L2 1.8e-3 / max |err|
# 3.2e-3 (`splade` style) and 4.6e-4 / 8.7e-4 (`hf`); one H100 measured 1.9e-3 / 3.4e-3 and 5.7e-4 / 1.2e-3.
REL_BAR = 4e-3
ABS_BAR = 1e-2
# Against the HF fp32 golden (tests/golden/splade_golden.npz), up to 12 layers: the head's fp16-operand floor per case
# (rel-L2, max |err| over the words the golden stores; measured on the CPU against the fp64 oracle, which matches HF to
# <= 1e-5), and the bars, about 2.5x and 3.5x the worst floor.
GOLDEN_FLOOR = {"base2_hf": (4.2e-4, 6.0e-4), "base2_splade": (1.8e-3, 2.9e-3), "base12_hf": (4.0e-4, 6.7e-4),
                "base12_splade": (4.1e-3, 4.2e-3), "small2_splade": (1.8e-3, 3.4e-3)}
GOLDEN_REL_BAR = 1e-2
GOLDEN_ABS_BAR = 1.5e-2


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _model(rt, g, flat):
    return rt.SparseEmbedModel(R.geometry_dict(g), SR.pack_splade_blob(flat, g))


def _device(rt, model, ids, lens, S=None):
    """b200rt_embed_device of the batch padded to S (default its own width) on replica 0."""
    import torch

    B, S0 = ids.shape
    S = S or S0
    pad = np.zeros((B, S), np.int32)
    pad[:, :S0] = ids
    d_ids = torch.from_numpy(pad).cuda()
    d_lens = torch.from_numpy(np.ascontiguousarray(lens, np.int32)).cuda()
    d_out = torch.empty((B, model.out_dim), dtype=torch.float32, device="cuda")
    model.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), B, S, d_out.data_ptr(), 0)
    rt.device_sync(0)
    return d_out.cpu().numpy()


# ================================================================================================ embedders are unchanged

@gpu
def test_embedder_and_reranker_beside_splade_are_unchanged(rt):
    """Runs first: a bge-base CLS embedder's vectors and a reranker's logits before any SPLADE model exists in the runtime, and
    again after one loaded and ran (whose head uses ctx, pstats[1] and ffn as scratch), bitwise the same."""
    g = R.BertGeometry(layers=2)
    flat = R.make_weights(g, 3, "trained")
    emb = rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g))
    ids, lens = FC.ragged_batch([192, 1, 64, 65, 130], 192, seed=17)
    cg = R.BertGeometry(layers=2, **GEOMS["small"])
    clf = rt.ClassifierModel(RR.geometry_dict(cg, 1), RR.pack_classifier_blob(RR.make_classifier_weights(cg, 1, "trained", 1), cg))
    pids, plens, psegs = RR.synth_pairs([50, 20], [30, 20], 64, 3)
    before, lbefore = emb.embed(ids, lens), clf.classify(pids, plens, psegs)
    sg = R.BertGeometry(layers=2)
    sp = _model(rt, sg, SR.make_splade_weights(sg, 2, "hf"))
    sp.embed(ids, lens)
    after, lafter = emb.embed(ids, lens), clf.classify(pids, plens, psegs)
    print(f"embedder / reranker before and after a SPLADE model: bitwise equal {np.array_equal(_bits(before), _bits(after))} / "
          f"{np.array_equal(_bits(lbefore), _bits(lafter))}")
    assert np.array_equal(_bits(before), _bits(after)) and np.array_equal(_bits(lbefore), _bits(lafter))


# ================================================================================================ kernels

def _splade_operands(rng, B, S, K, vocab):
    """u-like fp16 rows (gelu outputs: skewed, some large), their partials, a decoder and a bias with a share of columns that
    stay negative everywhere (their maxima must be exactly 0)."""
    x = rng.standard_normal((B * S, K))
    u = (x * (x > -0.5) * 1.3 + 0.2 * rng.standard_normal(K)).astype(np.float16)
    stats = KR.partials(u.astype(np.float64)).astype(np.float32)
    w = (rng.standard_normal((vocab, K)) * (1.0 / np.sqrt(K))).astype(np.float16)
    N = SR.vpad(vocab)
    c = (rng.standard_normal(N) - 1.0).astype(np.float32)
    c[rng.random(N) < 0.2] = -20.0
    return u, stats, w, c, N


@gpu
@pytest.mark.parametrize("K", [384, 768, 1024])
@pytest.mark.parametrize("S", [64, 512])
def test_gemm_splade_kernel(rt, K, S):
    rng = np.random.default_rng(K + S)
    lens = np.array([1, S, 63, 65, 127, 129], np.int32)
    vocab = 30522 if S == 64 else 1000  # the full vocabulary's last tile at S = 64; a narrower decoder keeps the 512 case cheap
    u, stats, w, c, N = _splade_operands(rng, len(lens), S, K, vocab)
    full, _ = rt.debug_gemm_splade(u, w, c, stats, lens, S, N, 1e-12)
    m = SR.check_gemm_splade(f"gemm_splade K={K} S={S} vocab={vocab}", full, u, w, c, stats, lens, S, 1e-12)
    assert m < 1
    nz = (full[:, :vocab] != 0).mean()
    print(f"  non-zero maxima {nz:.2f}")
    assert 0.2 < nz < 0.95
    for sms in (1, 7):
        o, _ = rt.debug_gemm_splade(u, w, c, stats, lens, S, N, 1e-12, sms=sms)
        assert np.array_equal(o, full), f"sms={sms} differs from every SM"


@gpu
@pytest.mark.parametrize("W", [384, 768, 1024])
def test_mlm_ln_stats_kernel(rt, W):
    rng = np.random.default_rng(W)
    u = (rng.standard_normal((301, W)) * 3.0 + rng.standard_normal(W)).astype(np.float16)
    st, vmax = rt.debug_mlm_ln_stats(u, n_max=4099)
    KR.check_partials(f"mlm_ln_stats W={W}", st, u.astype(np.float64))
    assert (vmax == 0).all(), "the max buffer was not zeroed"


@gpu
def test_splade_finalize_kernel(rt):
    bits = SR.finalize_probe()
    out = rt.debug_splade_finalize(bits, 500)
    assert SR.check_splade_finalize("splade_finalize", out, bits, 500) < 1
    assert (out[:, :][bits[:, :500] == 0] == 0).all()


# ================================================================================================ forward chain

class SpladeChain(FC.TextChain):
    """TextChain of a SPLADE encoder: the four head launches after the last layer.  With a row sample, `items` are the items
    whose maxima gemm_splade is checked on (a max reads every row of its item)."""

    def __init__(self, flat, g, ids, lens, fold, rows=None, items=None):
        super().__init__(flat, g, ids, lens, fold, rows)
        self.items = np.arange(self.B) if items is None else np.asarray(items)
        f, last = flat, f"l{g.layers - 1}.ln2."
        self.t16, self.tc = fold(f["mlm.t.w"], f[last + "g"], f[last + "b"], f["mlm.t.b"])
        self.dec16, dc = fold(f["mlm.dec.w"], f["mlm.ln.g"], f["mlm.ln.b"], f["mlm.dec.b"])
        self.vpad = SR.vpad(g.vocab)
        self.dc = np.zeros(self.vpad, np.float32)
        self.dc[: g.vocab] = dc

    def vmax(self, t):
        return np.ascontiguousarray(t["ffn"]).reshape(-1).view(np.uint32)[: self.B * self.vpad].reshape(self.B, self.vpad)

    def check(self, tag, name, l, prev, cur):
        g, what, rows = self.g, f"{tag} {name}", self.rows
        if name == "gemm_mlm_transform":
            return KR.check_gemm(what, cur["ctx"][rows], 1, prev["yhi"][rows], self.t16, self.tc, ln_stats=prev["pstats0"][rows], eps=g.eps)
        if name == "mlm_ln_stats":
            assert (self.vmax(cur) == 0).all(), f"{what}: max buffer not zeroed"
            return KR.check_partials(what, cur["pstats1"][rows], cur["ctx"][rows].astype(np.float64))
        if name == "gemm_splade":
            it = self.items
            item_rows = (it[:, None] * self.S + np.arange(self.S)).reshape(-1)
            return SR.check_gemm_splade(what, self.vmax(cur)[it], prev["ctx"][item_rows], self.dec16, self.dc, prev["pstats1"][item_rows],
                                        self.lens[it], self.S, g.eps)
        if name == "splade_finalize":
            return SR.check_splade_finalize(what, cur["out"], self.vmax(prev), g.vocab)
        return super().check(tag, name, l, prev, cur)


HEAD = ("gemm_mlm_transform", "mlm_ln_stats", "gemm_splade", "splade_finalize")


@pytest.fixture
def chain_names(monkeypatch):
    """run_chain's launch tables, extended by the SPLADE head.  mlm_ln_stats and gemm_splade use the start of ffn as a uint32
    [B, vpad] max buffer, whose words are no fp16 values: for them the ffn invariants are checked here, on those words (the
    buffer's rows past it unchanged, its guard rows still poison), and the generic checks run on the other buffers."""
    monkeypatch.setitem(FC.WRITES, "gemm_mlm_transform", ("ctx",))
    monkeypatch.setitem(FC.WRITES, "mlm_ln_stats", ("pstats1",))
    monkeypatch.setitem(FC.WRITES, "gemm_splade", ())
    monkeypatch.setitem(FC.WRITES, "splade_finalize", ())
    monkeypatch.setattr(FC, "POOLS", FC.POOLS + ("splade_finalize",))
    generic = FC.check_invariants

    def check_invariants(tag, name, prev, cur, ch):
        if name not in ("mlm_ln_stats", "gemm_splade"):
            return generic(tag, name, prev, cur, ch)
        n = ch.B * ch.vpad
        p = np.ascontiguousarray(prev["ffn"]).reshape(-1).view(np.uint32)
        c = np.ascontiguousarray(cur["ffn"]).reshape(-1).view(np.uint32)
        assert np.array_equal(p[n:], c[n:]), f"{tag}: {name} wrote ffn past its {ch.B} x {ch.vpad} maxima"
        generic(tag, name, prev, dict(cur, ffn=prev["ffn"]), ch)

    monkeypatch.setattr(FC, "check_invariants", check_invariants)


def _chain(rt, g, style, seed, lens, S):
    flat = SR.make_splade_weights(g, seed, style)
    model = _model(rt, g, flat)
    ids, lens = FC.ragged_batch(lens, S, seed=seed + 1)
    ch = SpladeChain(flat, g, ids, lens, FC.gpu_fold(rt))
    margins = {}
    last = FC.run_chain(f"splade {style}", ch, lambda k: model.debug_trace(ids, lens, k), margins)
    FC.print_margins(f"splade {style} hidden {g.hidden}", margins)
    assert last["names"][-4:] == list(HEAD) and last["n_total"] == 5 * g.layers + 5
    return flat, model, ids, lens, last


@gpu
@pytest.mark.parametrize("geometry,style", [("base", "splade"), ("small", "hf"), ("large", "splade")])
def test_splade_chain(rt, chain_names, geometry, style):
    """2 layers, 5 ragged items padded to 128 (one of one token, both sides of the 64-row half).  embed() (scheduler, buckets,
    graph replay) and the device-resident entry are bitwise the traced vectors, and one forward is 5 L + 5 launches."""
    g = R.BertGeometry(layers=2, **GEOMS[geometry])
    flat, model, ids, lens, last = _chain(rt, g, style, 5, [128, 1, 64, 65, 100], 128)
    traced = last["out"]
    for what, o in (("embed()", model.embed(ids, lens)), ("embed_device", _device(rt, model, ids, lens))):
        same = np.array_equal(_bits(o), _bits(traced))
        print(f"{what}: bitwise the traced vectors: {same}")
        assert same, what
    n0 = rt.stats()["kernel_launches"]
    model.embed(ids[:1], lens[:1])
    assert rt.stats()["kernel_launches"] - n0 == last["n_total"] + 1  # + the wave's scatter


@gpu
def test_splade_full_wave_chain(rt, chain_names):
    """One wave at capacity: debug_cap_rows() // 128 items of the 128-token bucket (528 on an H100 SXM), 2-layer bge-base
    geometry, `splade` weights; every launch checked on full_wave_chain's row sample, gemm_splade on every row and word of the
    first, second, middle and last items, splade_finalize on the whole wave.  embed() and the device entry are bitwise the
    traced vectors."""
    t0 = time.perf_counter()
    g = R.BertGeometry(layers=2)
    flat = SR.make_splade_weights(g, 8, "splade")
    model = _model(rt, g, flat)
    cap = model.debug_cap_rows()
    S = 128
    B = cap // S
    ids, lens = FC.ragged_batch(FW.ragged_lens(B, S, seed=51), S, seed=52)
    lens[[0, 1, B // 2, B - 1]] = [1, 64, 65, S]
    ids, lens = FC.ragged_batch(lens, S, seed=52)
    rows = FW.sample_rows(B, S)
    print(FW.coverage(rows, B, S))
    ch = SpladeChain(flat, g, ids, lens, FC.gpu_fold(rt), rows=rows, items=[0, 1, B // 2, B - 1])
    last = FW._run("splade full wave", ch, lambda k: model.debug_trace(ids, lens, k), cap, t0)
    assert np.array_equal(_bits(model.embed(ids, lens)), _bits(last["out"]))
    assert np.array_equal(_bits(_device(rt, model, ids, lens)), _bits(last["out"]))


# ================================================================================================ parity

@gpu
@pytest.mark.parametrize("style", ["hf", "splade"])
def test_parity_with_oracle(rt, style):
    """2-layer bge-base geometry, ragged items over the 64-512 buckets (1, 63, 64, 65, 127, 129, 300 and 512 tokens) against the
    fp64 oracle: per-item rel-L2 <= REL_BAR and max |err| <= ABS_BAR, the same support wherever the oracle is more than twice
    ABS_BAR from 0, and the same top-10 words wherever the oracle's 10th and 11th differ by more than twice ABS_BAR."""
    g = R.BertGeometry(layers=2)
    flat = SR.make_splade_weights(g, 21, style)
    model = _model(rt, g, flat)
    lens = [1, 63, 64, 65, 127, 129, 300, 512]
    ids, lens = FC.ragged_batch(lens, 512, seed=22)
    got = model.embed(ids, lens).astype(np.float64)
    ref = SR.splade_np(flat, ids, lens, g)
    floor = SR.splade_fp16_operands(flat, ids, lens, g)
    rel, err = R.rel_l2(got, ref), np.abs(got - ref).max(1)
    frel, ferr = R.rel_l2(floor, ref), np.abs(floor - ref).max(1)
    nnz = (ref > 0).sum(1)
    print(f"{style}: non-zero words per item {nnz.tolist()}")
    print(f"{style}: rel-L2 max {rel.max():.2e} (bar {REL_BAR:g}, head fp16-operand floor {frel.max():.2e}); max |err| {err.max():.2e} "
          f"(bar {ABS_BAR:g}, floor {ferr.max():.2e})")
    assert rel.max() <= REL_BAR and err.max() <= ABS_BAR
    sure = np.abs(ref) > 2 * ABS_BAR
    assert ((got > 0) == (ref > 0))[sure].all(), "support differs where the oracle is clearly non-zero"
    for i in range(len(lens)):
        o = np.sort(ref[i])[::-1]
        if o[9] - o[10] > 2 * ABS_BAR:
            assert set(np.argsort(-got[i])[:10]) == set(np.argsort(-ref[i])[:10]), f"item {i}: top-10 words differ"


@gpu
@pytest.mark.parametrize("name", list(msg.CASES))
def test_parity_with_hf_golden(rt, name):
    """Each golden case against HF fp32, over the words the golden stores (all of them for `splade` cases, a 544-word sample
    for the dense `hf` ones): per-item rel-L2 and max |err| within the bars, the same support wherever HF is more than twice
    the absolute bar away from 0, and the same top-10 words wherever HF's 10th and 11th are that far apart."""
    golden = np.load(os.path.join(GOLDEN, "splade_golden.npz"))
    ids, lens = golden["ids"], golden["lens"]
    g = msg.geometry(name)
    cols, ref = msg.reference(golden, name)
    got = _model(rt, g, msg.weights(name)).embed(ids, lens)[:, cols].astype(np.float64)
    ref = ref.astype(np.float64)
    rel, err = R.rel_l2(got, ref), np.abs(got - ref).max(1)
    fr, fa = GOLDEN_FLOOR[name]
    print(f"{name}: rel-L2 max {rel.max():.2e} (bar {GOLDEN_REL_BAR:g}, floor {fr:.1e}), max |err| {err.max():.2e} "
          f"(bar {GOLDEN_ABS_BAR:g}, floor {fa:.1e}); non-zero words GPU {(got > 0).sum(1).tolist()} HF {(ref > 0).sum(1).tolist()}")
    assert rel.max() <= GOLDEN_REL_BAR and err.max() <= GOLDEN_ABS_BAR
    sure = np.abs(ref) > 2 * GOLDEN_ABS_BAR
    assert ((got > 0) == (ref > 0))[sure].all()
    for i in range(len(lens)):
        o = np.sort(ref[i])[::-1]
        if o[9] - o[10] > 2 * GOLDEN_ABS_BAR:
            assert set(np.argsort(-got[i])[:10]) == set(np.argsort(-ref[i])[:10]), f"item {i}: top-10 words differ"


# ================================================================================================ invariance

@gpu
def test_vectors_invariant_across_batches_and_shapes(rt):
    """An item's vector, bitwise: alone, together, inside full waves of the 64- and the 512-token bucket (at the start, middle
    and end), padded to 128 and 512 through the device-resident entry, and through the trace."""
    g = R.BertGeometry(layers=2)
    model = _model(rt, g, SR.make_splade_weights(g, 7, "splade"))
    ids, lens = FC.ragged_batch([60, 1, 64, 33], 64, seed=9)
    alone = np.concatenate([model.embed(ids[i:i + 1], lens[i:i + 1]) for i in range(4)])
    assert np.array_equal(_bits(model.embed(ids, lens)), _bits(alone))
    cap = model.debug_cap_rows()
    for S in (64, 512):
        B = cap // S
        wl = np.random.default_rng(S).integers(S - 63, S + 1, size=B).astype(np.int32)
        wids, wl = FC.ragged_batch(wl, S, seed=S + 1)
        at = [0, B // 2 + 1, B - 4]
        for p in at:
            for k in range(4):
                wids[p + k] = 0
                wids[p + k, :64] = ids[k]
                wl[p + k] = lens[k]
        t0 = time.perf_counter()
        wave = model.embed(wids, wl)
        print(f"full wave {B} x {S}: {time.perf_counter() - t0:.2f} s")
        for p in at:
            assert np.array_equal(_bits(wave[p:p + 4]), _bits(alone)), f"{B} x {S} wave at item {p}"
    for S in (128, 512):
        assert np.array_equal(_bits(_device(rt, model, ids, lens, S)), _bits(alone)), f"padded to {S}"
    assert np.array_equal(_bits(model.debug_trace(ids, lens, 5 * g.layers + 5)["out"]), _bits(alone))


@gpu
def test_splade_refusals(rt):
    import b200rt

    g = R.BertGeometry(layers=1)
    model = _model(rt, g, SR.make_splade_weights(g, 1, "hf"))
    ids, lens = FC.ragged_batch([10, 20], 64, seed=1)
    with pytest.raises(b200rt.B200RTError) as e:
        model._submit(ids, lens, np.array([5, 5], np.int32), None, None, False)
    assert e.value.code == b200rt.E_INVALID
    with pytest.raises(b200rt.B200RTError) as e:
        _device(rt, model, ids[:, :40], lens, 40)
    assert e.value.code == b200rt.E_INVALID and "multiples of 64" in str(e.value)
    big = dict(R.geometry_dict(g), vocab=49153)
    with pytest.raises(b200rt.B200RTError) as e:
        b200rt.SparseEmbedModel(big, np.zeros(8, np.float32))
    assert e.value.code == b200rt.E_UNSUPPORTED


# ================================================================================================ router

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _post(port, path, body):
    req = urllib.request.Request(f"http://127.0.0.1:{port}{path}", data=json.dumps(body).encode(),
                                 headers={"Content-Type": "application/json"})
    try:
        with urllib.request.urlopen(req, timeout=120) as r:
            return r.status, json.loads(r.read())
    except urllib.error.HTTPError as e:
        return e.code, json.loads(e.read())


@gpu
def test_router_embed_sparse(tmp_path):
    """text-embeddings-router --pooling splade on a BertForMaskedLM snapshot (config.json + model.safetensors without
    decoder.weight, as tied checkpoints are saved): /embed_sparse against the oracle, /info, and the 400 on /embed."""
    from b200rt import weights as W
    from tei_router.tokenizer import WordPiece

    g = R.BertGeometry(layers=2)
    flat = SR.make_splade_weights(g, 31, "splade")
    snap = tmp_path / "snap"
    snap.mkdir()
    sd = {"bert." + k: v for k, v in R.flat_to_hf_state({k: v for k, v in flat.items() if not k.startswith("mlm.")}, g).items()}
    t = "cls.predictions.transform."
    sd.update({t + "dense.weight": flat["mlm.t.w"], t + "dense.bias": flat["mlm.t.b"], t + "LayerNorm.weight": flat["mlm.ln.g"],
               t + "LayerNorm.bias": flat["mlm.ln.b"], "cls.predictions.bias": flat["mlm.dec.b"]})
    W.write_safetensors(str(snap / "model.safetensors"), {k: np.ascontiguousarray(v, np.float32) for k, v in sd.items()})
    (snap / "config.json").write_text(json.dumps({"architectures": ["BertForMaskedLM"], "layer_norm_eps": 1e-12,
                                                  "num_attention_heads": 12}))
    port = _free_port()
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    proc = subprocess.Popen([os.sys.executable, "-m", "tei_router.server", "--model-id", "local/splade", "--pooling", "splade",
                             "--weights", str(snap), "--port", str(port), "--gpus", "1"], cwd=PKG, env=env,
                            stderr=subprocess.PIPE, text=True)
    try:
        for _ in range(600):
            try:
                with socket.create_connection(("127.0.0.1", port), timeout=1):
                    break
            except OSError:
                assert proc.poll() is None, proc.stderr.read()
                time.sleep(0.5)
        texts = ["a short query", "sparse retrieval with learned term weights " * 5]
        code, body = _post(port, "/embed_sparse", {"inputs": texts})
        assert code == 200 and len(body) == 2
        tok = WordPiece(None)
        rows = [tok.encode(x, 512, True) for x in texts]
        lens = np.array([len(r) for r in rows], np.int32)
        ids = np.zeros((2, lens.max()), np.int32)
        for i, r in enumerate(rows):
            ids[i, : len(r)] = r
        ref = SR.splade_np(flat, ids, lens, g)
        for i, sparse in enumerate(body):
            idx = [e["index"] for e in sparse]
            assert idx == sorted(idx) and all(e["value"] > 0 for e in sparse)
            dense = np.zeros(g.vocab)
            dense[idx] = [e["value"] for e in sparse]
            print(f"router item {i}: {len(idx)} words, rel-L2 vs oracle {R.rel_l2(dense[None], ref[i:i + 1])[0]:.2e}")
            assert R.rel_l2(dense[None], ref[i:i + 1])[0] <= REL_BAR
        code, single = _post(port, "/embed_sparse", {"inputs": texts[0]})
        assert code == 200 and single == body[:1]
        assert _post(port, "/embed", {"inputs": "x"})[0] == 400
        assert _post(port, "/embed_sparse", {"input": "x"})[0] == 422
        with urllib.request.urlopen(f"http://127.0.0.1:{port}/info", timeout=30) as r:
            assert json.loads(r.read())["pooling"] == "splade"
    finally:
        proc.terminate()
        proc.wait(timeout=60)
