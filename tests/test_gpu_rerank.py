"""GPU: BERT cross-encoders / sequence classifiers (kind "bert_classifier") -- the two kernels the classifier path adds, the
whole forward launch by launch, parity with HF fp32, bitwise invariance of an item's logits, and the router's /rerank and
/predict.

  * kernels: embed_kernel with segments bit for bit against numpy; cls_head_kernel against its fp64 reference at W = 384 /
    768 / 1024 and L = 1, 2, 64, and bitwise the same on one block as on one block per item;
  * forward chain: a 2-layer classifier on a ragged pair batch through run_chain (tests/test_gpu_forward_chain.py) with a
    TextChain subclass that checks `embed` with segments and `cls_head`, then one full wave (debug_cap_rows() // 256 pairs,
    the row sample of tests/test_gpu_full_wave_chain.py); submit_pairs, the device-resident entry and the trace agree bitwise;
  * parity: the golden's HF fp32 logits (tests/golden/rerank_golden.npz) within PARITY_BAR of the logits' spread, and the
    GPU ranks two texts as the oracle does wherever the oracle's scores differ by more than twice the bar;
  * invariance: an item's logits are bitwise the same alone, inside a batch of a full wave's items and at another padded
    length; an embedding model loaded beside the classifier is bitwise unchanged."""
import importlib.util
import json
import os
import socket
import subprocess
import time
import urllib.error
import urllib.request

import numpy as np
import pytest

import kernel_refs as KR
import rerank_refs as RR
import test_gpu_forward_chain as FC
import test_gpu_full_wave_chain as FW
from oracle import bge_ref as R

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "modal-examples_b200")
GOLDEN = os.path.join(ROOT, "tests", "golden")
_spec = importlib.util.spec_from_file_location("make_rerank_golden", os.path.join(GOLDEN, "make_rerank_golden.py"))
mrg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mrg)

# Parity bar: max |GPU - HF fp32| over the batch, as a fraction of the logits' spread (max - min).  Its floor is what the fp16
# operands alone cost (rerank_refs.classify_fp16_operands against the fp64 oracle on the golden batch, measured on the CPU):
FLOOR = {"l6_hf": 3.2e-4, "l6_trained": 1.4e-4, "l12_hf": 4.6e-4, "l12_trained": 1.3e-4, "base2_trained": 9.0e-5}
PARITY_BAR = 2e-3  # about 4x the worst floor (12 layers, HF init, whose logits span only ~0.1)

MINILM = dict(hidden=384, heads=12, inter=1536)


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _classifier(rt, g, flat):
    return rt.ClassifierModel(RR.geometry_dict(g, flat["cls.w"].shape[0]), RR.pack_classifier_blob(flat, g))


def _device(rt, model, ids, lens, segs, S=None):
    """b200rt_embed_device_pairs of the batch padded to S (default its own width) on replica 0."""
    import torch

    B, S0 = ids.shape
    S = S or S0
    pad = np.zeros((B, S), np.int32)
    pad[:, :S0] = ids
    d_ids = torch.from_numpy(pad).cuda()
    d_lens = torch.from_numpy(np.ascontiguousarray(lens, np.int32)).cuda()
    d_segs = torch.from_numpy(np.ascontiguousarray(segs, np.int32)).cuda() if segs is not None else None
    d_out = torch.empty((B, model.out_dim), dtype=torch.float32, device="cuda")
    model.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), B, S, d_out.data_ptr(), 0, d_segs.data_ptr() if d_segs is not None else 0)
    rt.device_sync(0)
    return d_out.cpu().numpy()


# ================================================================================================ embedders are unchanged

@gpu
def test_embedder_beside_classifier_is_unchanged(rt):
    """Runs first: a bge-base embedder's vectors before any classifier exists in the runtime, and again after a classifier
    loaded and ran (which allocates the segment buffers), bitwise the same -- through the scheduler and embed_device."""
    g = R.BertGeometry(layers=2)
    flat = R.make_weights(g, 3, "trained")
    emb = rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g))
    ids, lens = FC.ragged_batch([192, 1, 64, 65, 130], 192, seed=17)
    before = emb.embed(ids, lens)
    import torch

    d_ids, d_lens = torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda()
    d_out = torch.empty((5, 768), dtype=torch.float32, device="cuda")
    emb.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), 5, 192, d_out.data_ptr(), 0)
    rt.device_sync(0)
    dev_before = d_out.cpu().numpy()
    cg = R.BertGeometry(layers=2, **MINILM)
    clf = _classifier(rt, cg, RR.make_classifier_weights(cg, 1, "trained", 1))
    pids, plens, psegs = RR.synth_pairs([50, 20], [30, 20], 64, 3)
    clf.classify(pids, plens, psegs)
    after = emb.embed(ids, lens)
    emb.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), 5, 192, d_out.data_ptr(), 0)
    rt.device_sync(0)
    print(f"bge-base embed() before / after a classifier: bitwise equal {np.array_equal(_bits(before), _bits(after))}")
    assert np.array_equal(_bits(before), _bits(after))
    assert np.array_equal(_bits(dev_before), _bits(d_out.cpu().numpy()))
    assert np.array_equal(_bits(before), _bits(dev_before))


# ================================================================================================ kernels

@gpu
@pytest.mark.parametrize("W", [384, 768, 1024])
def test_embed_segs_bit_exact(rt, W):
    """embed with segments, bit for bit, including segment starts outside [0, S] (clamped on the device) and the two ends."""
    rng = np.random.default_rng(W)
    B, S, vocab = 8, 96, 2000
    word = rng.standard_normal((vocab, W), dtype=np.float32)
    pos = rng.standard_normal((S, W), dtype=np.float32)
    type2 = rng.standard_normal((2, W), dtype=np.float32)
    ids = rng.integers(0, vocab, size=B * S).astype(np.int32)
    segs = np.array([0, 1, 40, S - 1, S, -3, S + 7, 64], np.int32)
    hi, lo, st = rt.debug_embed_segs(ids, segs, word, pos, type2, S, hidden=W)
    RR.check_embed_segs(f"embed segs W={W}", hi, lo, st, ids, segs, word, pos, type2, S)
    # without segments the type row is 0 everywhere: the existing entry, same bits as segs = S
    hi0, lo0, _ = rt.debug_embed(ids, word, pos, type2[0], S, hidden=W)
    his, los, _ = rt.debug_embed_segs(ids, np.full(B, S, np.int32), word, pos, type2, S, hidden=W)
    assert np.array_equal(hi0.view(np.uint16), his.view(np.uint16)) and np.array_equal(lo0.view(np.uint16), los.view(np.uint16))


@gpu
@pytest.mark.parametrize("W", [384, 768, 1024])
@pytest.mark.parametrize("L", [1, 2, 64])
def test_cls_head_kernel(rt, W, L):
    """cls_head against its fp64 reference (named roundings: the LayerNorm's, each dot product's fp32 chain, tanhf), and
    bitwise the same on 1 block, 7 blocks and one block per item."""
    rng = np.random.default_rng(W + L)
    B, S = 37, 5
    x = (rng.standard_normal((B * S, W)) * 2.0 + rng.standard_normal(W)).astype(np.float32)
    hi, lo = KR.split_hilo(x)
    gamma = (1.0 + 0.1 * rng.standard_normal(W)).astype(np.float32)
    beta = (0.05 * rng.standard_normal(W)).astype(np.float32)
    pw = (rng.standard_normal((W, W)) * 1.5 / np.sqrt(W)).astype(np.float32)
    pb = (0.1 * rng.standard_normal(W)).astype(np.float32)
    cw = (rng.standard_normal((L, W)) * 0.3).astype(np.float32)
    cb = rng.standard_normal(L).astype(np.float32)
    full = rt.debug_cls_head(hi, lo, gamma, beta, pw, pb, cw, cb, S, 1e-12, hidden=W)
    m = RR.check_cls_head(f"cls_head W={W} L={L}", full, hi, lo, gamma, beta, pw, pb, cw, cb, S, 1e-12)
    assert m < 1
    for ctas in (1, 7):
        o = rt.debug_cls_head(hi, lo, gamma, beta, pw, pb, cw, cb, S, 1e-12, hidden=W, ctas=ctas)
        assert np.array_equal(_bits(o), _bits(full)), f"{ctas} blocks differ from one block per item"


# ================================================================================================ forward chain

class ClassifierChain(FC.TextChain):
    """TextChain of a BERT classifier: `embed` with the batch's segment starts and the `cls_head` launch in place of a pool."""

    def __init__(self, flat, g, ids, lens, segs, fold, rows=None):
        super().__init__(flat, g, ids, lens, fold, rows)
        self.segs = np.asarray(segs, np.int32)

    def check(self, tag, name, l, prev, cur):
        f, M, what = self.flat, self.M, f"{tag} layer {l} {name}"
        if name == "embed":
            return RR.check_embed_segs(what, cur["yhi"][:M], cur["ylo"][:M], cur["pstats0"][self.rows], self.ids.reshape(-1), self.segs,
                                       f["emb.word"], f["emb.pos"], f["emb.type"], self.S, rows=self.rows)
        if name == "cls_head":
            last = f"l{self.g.layers - 1}.ln2."
            return RR.check_cls_head(what, cur["out"], prev["yhi"][:M], prev["ylo"][:M], f[last + "g"], f[last + "b"], f["pool.w"],
                                     f["pool.b"], f["cls.w"], f["cls.b"], self.S, self.g.eps)
        return super().check(tag, name, l, prev, cur)


@pytest.fixture
def chain_names(monkeypatch):
    """run_chain's launch tables, extended by the classifier's last launch (which writes only `out`)."""
    monkeypatch.setitem(FC.WRITES, "cls_head", ())
    monkeypatch.setattr(FC, "POOLS", FC.POOLS + ("cls_head",))


LENS, SEGS, S_CHAIN = [192, 3, 64, 65, 130, 1], [100, 2, 63, 65, 20, 1], 192


@gpu
@pytest.mark.parametrize("geometry,L", [("small", 1), ("base", 2)])
def test_classifier_chain(rt, chain_names, geometry, L):
    """2 layers, 6 ragged pairs padded to 192 (a second segment of one token, an empty first text, single sequences, an item
    of one token).  Then classify() (scheduler, buckets, graph replay), the device-resident entry and the trace agree bitwise,
    and one forward is 5 L + 2 launches."""
    g = R.BertGeometry(layers=2, **(MINILM if geometry == "small" else {}))
    flat = RR.make_classifier_weights(g, 5, "trained", L)
    model = _classifier(rt, g, flat)
    ids, lens, segs = RR.synth_pairs(LENS, SEGS, S_CHAIN, 31)
    ch = ClassifierChain(flat, g, ids, lens, segs, FC.gpu_fold(rt))
    margins = {}
    last = FC.run_chain(f"classifier {geometry} L={L}", ch, lambda k: model.debug_trace(ids, lens, k, segs=segs), margins)
    FC.print_margins(f"classifier {geometry} L={L}", margins)
    assert last["names"][-1] == "cls_head" and last["n_total"] == 5 * g.layers + 2
    traced = last["out"]
    sched = model.classify(ids, lens, segs)
    dev = _device(rt, model, ids, lens, segs)
    for what, o in (("classify()", sched), ("embed_device_pairs", dev)):
        same = np.array_equal(_bits(o), _bits(traced))
        print(f"{what}: bitwise the traced logits: {same}")
        assert same, what
    n0 = rt.stats()["kernel_launches"]
    model.classify(ids[:1], lens[:1], segs[:1])
    assert rt.stats()["kernel_launches"] - n0 == last["n_total"] + 1  # + the wave's scatter
    # the segments matter: the same ids as single sequences give other logits (except the single-sequence items)
    single = model.classify(ids, lens)
    assert not np.array_equal(_bits(single[0]), _bits(sched[0])) and np.array_equal(_bits(single[3]), _bits(sched[3]))


@gpu
def test_classifier_full_wave_chain(rt, chain_names):
    """One wave at capacity: debug_cap_rows() // 256 pairs of 256 tokens (where query + passage pairs land), 2-layer MiniLM
    geometry, every launch checked on full_wave_chain's row sample; the scheduler's and the device entry's logits are bitwise
    the traced ones."""
    t0 = time.perf_counter()
    g = R.BertGeometry(layers=2, **MINILM)
    flat = RR.make_classifier_weights(g, 6, "trained", 1)
    model = _classifier(rt, g, flat)
    cap = model.debug_cap_rows()
    S = 256
    B = cap // S
    lens = FW.ragged_lens(B, S, seed=41)
    rng = np.random.default_rng(42)
    segs = np.array([int(rng.integers(min(2, n), n + 1)) for n in lens], np.int32)
    segs[:3] = [lens[0], max(lens[1] - 1, 0), min(2, lens[2])]
    ids, lens, segs = RR.synth_pairs(lens, segs, S, 43)
    rows = FW.sample_rows(B, S)
    print(FW.coverage(rows, B, S))
    ch = ClassifierChain(flat, g, ids, lens, segs, FC.gpu_fold(rt), rows=rows)
    last = FW._run("classifier full wave", ch, lambda k: model.debug_trace(ids, lens, k, segs=segs), cap, t0)
    assert np.array_equal(_bits(model.classify(ids, lens, segs)), _bits(last["out"]))
    assert np.array_equal(_bits(_device(rt, model, ids, lens, segs)), _bits(last["out"]))


# ================================================================================================ parity

@gpu
@pytest.mark.parametrize("name", list(mrg.CASES))
def test_parity_with_hf_golden(rt, name):
    golden = np.load(os.path.join(GOLDEN, "rerank_golden.npz"))
    ids, lens, segs = golden["ids"], golden["lens"], golden["segs"]
    g, flat = mrg.geometry(name), mrg.weights(name)
    model = _classifier(rt, g, flat)
    got = model.classify(ids, lens, segs)
    ref = golden[f"{name}_logits"].astype(np.float64)
    spread = float(ref.max() - ref.min())
    err = float(np.abs(got - ref).max()) / spread
    print(f"{name}: GPU vs HF fp32 max |err| / spread = {err:.2e} (bar {PARITY_BAR:g}, fp16-operand floor {FLOOR[name]:.1e}, "
          f"spread {spread:.3g})")
    assert err < PARITY_BAR
    # rank agreement: any two items whose oracle scores differ by more than twice the bar are ordered the same way
    for j in range(ref.shape[1]):
        r, gq = ref[:, j], got[:, j].astype(np.float64)
        d = r[:, None] - r[None, :]
        sure = np.abs(d) > 2 * PARITY_BAR * spread
        agree = np.sign(gq[:, None] - gq[None, :]) == np.sign(d)
        print(f"{name} label {j}: {int(sure.sum()) // 2} ordered pairs decided, all agree: {bool(agree[sure].all())}")
        assert agree[sure].all()


# ================================================================================================ invariance

@gpu
def test_logits_invariant_across_batches_and_shapes(rt):
    """An item's logits, bitwise: alone, together, inside a batch of a full wave's items (at its start, middle and end; each
    item travels in its own length bucket with that batch's items of the bucket), padded to 256 and to 512 tokens through the
    device-resident entry, and through the trace.  With more than one replica in the pool the wave's items are spread over
    them, so the three positions land on different replicas."""
    g = R.BertGeometry(layers=6, **MINILM)
    flat = RR.make_classifier_weights(g, 11, "trained", 1)
    model = _classifier(rt, g, flat)
    ids, lens, segs = RR.synth_pairs([150, 40, 200, 3], [90, 39, 200, 2], 200, 5)
    alone = np.concatenate([model.classify(ids[i:i + 1], lens[i:i + 1], segs[i:i + 1]) for i in range(4)])
    together = model.classify(ids, lens, segs)
    assert np.array_equal(_bits(alone), _bits(together))
    B = model.debug_cap_rows() // 256
    wl = np.random.default_rng(1).integers(129, 257, size=B).astype(np.int32)
    ws = np.maximum(wl // 2, 2).astype(np.int32)
    wids, wl, ws = RR.synth_pairs(wl, ws, 256, 7)
    at = [0, B // 2 + 1, B - 4]
    for i, p in enumerate(at):
        for k in range(4):
            wids[p + k] = 0
            wids[p + k, :200] = ids[k]
            wl[p + k], ws[p + k] = lens[k], segs[k]
    wave = model.classify(wids, wl, ws)
    for p in at:
        assert np.array_equal(_bits(wave[p:p + 4]), _bits(alone)), f"full wave at item {p}"
    for S in (256, 512):
        assert np.array_equal(_bits(_device(rt, model, ids, lens, segs, S)), _bits(alone)), f"padded to {S}"
    assert np.array_equal(_bits(model.debug_trace(ids, lens, 5 * g.layers + 2, segs=segs)["out"]), _bits(alone))
    print(f"item logits bitwise equal alone, in a {B}-item batch at items {at}, padded to 256 / 512, traced "
          f"({rt.num_gpus()} replica(s) in the pool)")


# ================================================================================================ router

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _post(port, payload, path):
    req = urllib.request.Request(f"http://127.0.0.1:{port}{path}", data=json.dumps(payload).encode(), headers={"Content-Type": "application/json"})
    try:
        with urllib.request.urlopen(req, timeout=120) as r:
            return r.status, json.loads(r.read())
    except urllib.error.HTTPError as e:
        return e.code, json.loads(e.read())


def _get(port, path):
    with urllib.request.urlopen(f"http://127.0.0.1:{port}{path}", timeout=60) as r:
        return json.loads(r.read())


ROUTER_SEED = 17


@pytest.fixture(scope="module")
def reranker(tmp_path_factory):
    """text-embeddings-router --model-id cross-encoder/ms-marco-MiniLM-L-6-v2 with `trained` seeded weights as a flat blob."""
    g = R.BertGeometry(layers=6, **MINILM)
    flat = RR.make_classifier_weights(g, ROUTER_SEED, "trained", 1)
    path = tmp_path_factory.mktemp("w") / "reranker.bin"
    RR.pack_classifier_blob(flat, g).tofile(str(path))
    from tei_router.tokenizer import synthetic_vocab

    vocab = path.parent / "vocab.txt"  # a vocabulary file, so that the router does not switch auto-truncate on
    vocab.write_text("\n".join(synthetic_vocab()) + "\n")
    port = _free_port()
    env = dict(os.environ, PATH=os.path.join(PKG, "bin") + os.pathsep + os.environ["PATH"], B200RT_GPUS="1")
    proc = subprocess.Popen(["text-embeddings-router", "--model-id", "cross-encoder/ms-marco-MiniLM-L-6-v2", "--port", str(port),
                             "--weights", str(path), "--max-client-batch-size", "16", "--tokenizer-vocab", str(vocab)], env=env)
    deadline = time.time() + 300
    while True:
        try:
            socket.create_connection(("127.0.0.1", port), timeout=1).close()
            break
        except (socket.timeout, ConnectionRefusedError, OSError):
            assert proc.poll() is None, f"launcher exited unexpectedly with code {proc.returncode}"
            assert time.time() < deadline, "router did not become ready"
            time.sleep(0.2)
    yield port, g, flat
    proc.terminate()
    proc.wait(timeout=60)


def _oracle_pairs(pairs, truncate=False):
    from tei_router.tokenizer import WordPiece, synthetic_vocab

    tok = WordPiece({t: i for i, t in enumerate(synthetic_vocab())})
    rows = [tok.encode_pair(a, b, 512, truncate) if isinstance(b, str) else (tok.encode(a, 512, truncate), None) for a, b in pairs]
    lens = np.array([len(r) for r, _ in rows], np.int32)
    segs = np.array([s if s is not None else len(r) for r, s in rows], np.int32)
    ids = np.zeros((len(rows), int(lens.max())), np.int32)
    for i, (r, _) in enumerate(rows):
        ids[i, :len(r)] = r
    return ids, lens, segs


@gpu
def test_router_rerank_and_predict(reranker):
    port, g, flat = reranker
    info = _get(port, "/info")
    assert info["model_type"] == {"reranker": {"id2label": {"0": "LABEL_0"}, "label2id": {"LABEL_0": 0}}} and "pooling" not in info
    query = "what does a cross-encoder rerank?"
    texts = [f"passage {i}: {'retrieval ' * (i % 5)}ranks candidates {'by relevance ' * (i % 3)}for query #{i}" for i in range(12)]
    status, out = _post(port, {"query": query, "texts": texts, "raw_scores": True, "return_text": True}, "/rerank")
    assert status == 200 and len(out) == 12
    ids, lens, segs = _oracle_pairs([(query, t) for t in texts])
    ref = RR.classify_np(flat, ids, lens, segs, g)[:, 0]
    spread = float(ref.max() - ref.min())
    got = np.zeros(12)
    for r in out:
        got[r["index"]] = r["score"]
        assert r["text"] == texts[r["index"]]
    assert [r["score"] for r in out] == sorted(got, reverse=True)
    err = float(np.abs(got - ref).max()) / spread
    print(f"/rerank raw scores vs oracle: max |err| / spread = {err:.2e} (bar {PARITY_BAR:g}, spread {spread:.3g})")
    assert err < PARITY_BAR
    status, out2 = _post(port, {"query": query, "texts": texts}, "/rerank")
    sig = {r["index"]: r["score"] for r in out2}
    assert status == 200 and all(abs(sig[i] - 1 / (1 + np.exp(-ref[i]))) < PARITY_BAR * spread / 4 for i in range(12))
    assert "text" not in out2[0]
    # /predict: a pair, a batch of a pair and a single text; one label -> sigmoid
    status, p = _post(port, {"inputs": [query, texts[0]]}, "/predict")
    assert status == 200 and p[0]["label"] == "LABEL_0" and abs(p[0]["score"] - sig[0]) < 1e-6
    status, pb = _post(port, {"inputs": [[query, texts[1]], texts[2]], "raw_scores": True}, "/predict")
    ids2, lens2, segs2 = _oracle_pairs([(query, texts[1]), (texts[2], None)])
    ref2 = RR.classify_np(flat, ids2, lens2, segs2, g)[:, 0]
    assert status == 200 and len(pb) == 2
    assert all(abs(pb[i][0]["score"] - ref2[i]) < PARITY_BAR * spread for i in range(2))
    # refusals
    assert _post(port, {"inputs": ["a"]}, "/embed")[0] == 400
    assert _post(port, {"query": query, "texts": texts + texts}, "/rerank")[0] == 413  # > --max-client-batch-size 16
    long = "word " * 600
    assert _post(port, {"query": query, "texts": [long]}, "/rerank")[0] == 413
    status, out3 = _post(port, {"query": query, "texts": [long], "truncate": True, "raw_scores": True}, "/rerank")
    ids3, lens3, segs3 = _oracle_pairs([(query, long)], truncate=True)
    assert status == 200 and lens3[0] == 512
    assert abs(out3[0]["score"] - RR.classify_np(flat, ids3, lens3, segs3, g)[0, 0]) < PARITY_BAR * spread
    assert _post(port, {"query": 3, "texts": texts}, "/rerank")[0] == 422
