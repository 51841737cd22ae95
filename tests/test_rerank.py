"""CPU: BERT cross-encoders / sequence classifiers -- the oracle against HF and its golden, the `trained` head's statistics,
pair tokenisation against the Rust tokenizers, the classifier blob and its loaders, the router's host-side scoring, and the
kernel references of the classifier path (embed with token types, the pooler / classifier head) against numpy emulations
of the kernels and the mutants they must reject."""
import ctypes
import importlib.util
import json
import os

import numpy as np
import pytest

import kernel_refs as KR
import rerank_refs as RR
from oracle import bge_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

_spec = importlib.util.spec_from_file_location("make_rerank_golden", os.path.join(GOLDEN, "make_rerank_golden.py"))
mrg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mrg)

# The oracle restates HF; they agree to this fraction of the logits' spread (max - min over the batch).
HF_BAR = 5e-6

_weights = {}


def _case(name):
    if name not in _weights:
        _weights[name] = (mrg.geometry(name), mrg.weights(name))
    return _weights[name]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "rerank_golden.npz"))


# ================================================================================================ oracle

@pytest.mark.parametrize("name", list(mrg.CASES))
def test_oracle_matches_golden(golden, name):
    """classify_np (fp64) against HF BertForSequenceClassification fp32 as the golden recorded it."""
    g, flat = _case(name)
    ids, lens, segs = golden["ids"], golden["lens"], golden["segs"]
    assert np.array_equal(ids, mrg.inputs()[0]) and np.array_equal(segs, mrg.inputs()[2])
    ref = RR.classify_np(flat, ids, lens, segs, g)
    hf = golden[f"{name}_logits"]
    spread = float(ref.max() - ref.min())
    err = float(np.abs(hf - ref).max()) / spread
    print(f"{name}: oracle vs HF golden max |err| / spread = {err:.2e} (spread {spread:.3g}, bar {HF_BAR:g})")
    assert err < HF_BAR


def test_oracle_matches_hf_live():
    """A fresh HF model on a different batch (2 layers, bge-small geometry, 3 labels), token types included: the type row
    matters -- the same ids as single sequences give other logits."""
    g = R.BertGeometry(layers=2, hidden=384, heads=12, inter=1536)
    flat = RR.make_classifier_weights(g, 5, "trained", 3)
    ids, lens, segs = RR.synth_pairs([40, 9, 77, 5], [20, 3, 70, 5], 80, 4)
    hf = RR.classify_hf(RR.build_hf_classifier(flat, g), ids, lens, segs)
    ref = RR.classify_np(flat, ids, lens, segs, g)
    spread = float(ref.max() - ref.min())
    assert np.abs(hf - ref).max() / spread < HF_BAR
    single = RR.classify_np(flat, ids, lens, lens, g)
    assert np.abs(single[:3] - ref[:3]).max() > 1e-2 * spread  # item 3 is a single sequence either way
    assert np.array_equal(single[3], ref[3])


def test_hf_head_weights_match_random_classifier_blob():
    """The `hf` style is b200rt.weights.random_classifier_blob bit for bit, and its encoder prefix is random_blob's."""
    from b200rt import weights as W

    g = R.BertGeometry(layers=2, hidden=384, heads=12, inter=1536)
    gd = RR.geometry_dict(g, 2)
    blob = W.random_classifier_blob(gd, 9)
    assert np.array_equal(blob.view(np.uint32), RR.pack_classifier_blob(RR.make_classifier_weights(g, 9, "hf", 2), g).view(np.uint32))
    enc = W.random_blob(gd, 9)
    assert np.array_equal(blob[: enc.size].view(np.uint32), enc.view(np.uint32))
    # `trained`: the encoder is make_weights' own, unchanged by the head's draws
    tr = RR.make_classifier_weights(g, 9, "trained", 2)
    ref = R.make_weights(g, 9, "trained")
    assert all(np.array_equal(tr[k], ref[k]) for k in ref)


def test_trained_head_statistics(golden):
    """`trained`: the pooler's pre-activations at sigma ~1.5 with a sizeable share past |2| (tanh saturating), and logits
    spread over about +-10 -- on the golden batch, not the calibration batch the classifier was fitted to."""
    ids, lens, segs = golden["ids"], golden["lens"], golden["segs"]
    for name in ("l6_trained", "l12_trained", "base2_trained"):
        g, flat = _case(name)
        pre = RR.pooler_preactivations(flat, ids, lens, segs, g)
        z = RR.classify_np(flat, ids, lens, segs, g)
        sat = float((np.abs(pre) > 2.0).mean())
        print(f"{name}: pre-activation sigma {pre.std():.2f}, |pre| > 2 for {sat * 100:.0f} %, logits in [{z.min():.2f}, {z.max():.2f}], "
              f"sigma {z.std(0)}")
        assert 1.2 < pre.std() < 1.8 and sat > 0.08
        assert 4.0 < np.abs(z).max() < 15.0 and (z.std(0) > 1.0).all()
        assert z.max() - z.min() > 10.0
    for name in ("l6_hf", "l12_hf"):  # what the trained style is for: HF init leaves the tanh linear and the logits ~1e-1
        g, flat = _case(name)
        assert RR.pooler_preactivations(flat, ids, lens, segs, g).std() < 0.6
        assert np.abs(golden[f"{name}_logits"]).max() < 0.5


# ================================================================================================ tokenisation

@pytest.fixture(scope="module")
def fast_tok(tmp_path_factory):
    from transformers import BertTokenizerFast

    from tei_router.tokenizer import synthetic_vocab

    d = tmp_path_factory.mktemp("vocab")
    (d / "vocab.txt").write_text("\n".join(synthetic_vocab()) + "\n")
    return BertTokenizerFast(str(d / "vocab.txt"), do_lower_case=True)


def _words(rng, n):
    words = "the quick brown fox jumps over lazy dog retrieval ranking passage query neural search Zürich co-op 42".split()
    return " ".join(words[int(i)] for i in rng.integers(0, len(words), size=n))


def test_encode_pair_matches_fast_tokenizer(fast_tok):
    """[CLS] a [SEP] b [SEP] and its type ids as BertTokenizerFast (the Rust tokenizers TEI runs) gives them: short pairs,
    long ones, both texts too long, each text longer than the other, with longest_first truncation to many lengths.
    Both texts are non-empty: transformers' Python wrapper drops an empty second text and encodes a single sequence, which
    TEI (calling the Rust tokenizer with a pair) does not."""
    from tei_router.tokenizer import WordPiece

    wp = WordPiece()
    rng = np.random.default_rng(0)
    n_trunc = 0
    for _ in range(600):
        a, b = _words(rng, int(rng.integers(1, 60))), _words(rng, int(rng.integers(1, 60)))
        n = int(rng.integers(3, 130))
        enc = fast_tok(a, b, truncation="longest_first", max_length=n)
        ids, seg = wp.encode_pair(a, b, n, truncate=True)
        tt = enc["token_type_ids"]
        assert ids == enc["input_ids"], (a, b, n)
        assert seg == (tt.index(1) if 1 in tt else len(tt))
        full = fast_tok(a, b)["input_ids"]
        if len(full) > n:
            n_trunc += 1
            with pytest.raises(ValueError):
                wp.encode_pair(a, b, n, truncate=False)
        else:
            assert wp.encode_pair(a, b, n)[0] == full
    assert n_trunc > 200


def test_encode_pair_both_too_long():
    from tei_router.tokenizer import WordPiece

    wp = WordPiece()
    a, b = "alpha " * 300, "beta " * 280
    ids, seg = wp.encode_pair(a, b, 512, truncate=True)
    assert len(ids) == 512 and ids[seg - 1] == wp.sep and ids[-1] == wp.sep and ids[0] == wp.cls
    # m = 509 tokens for the texts: each gets 254, the longer (a) the odd one
    assert seg == 1 + 255 + 1


# ================================================================================================ weights and loaders

def test_classifier_blob_layout():
    from b200rt import weights as W

    g = dict(W.MS_MARCO_MINILM_L6_GEOMETRY)
    lay = W.classifier_blob_layout(g)
    assert lay[: len(W.blob_layout(g))] == W.blob_layout(g)
    assert lay[len(W.blob_layout(g)):] == [("pool.w", (384, 384)), ("pool.b", (384,)), ("cls.w", (1, 384)), ("cls.b", (128,))]
    assert all(int(np.prod(s)) % 128 == 0 for _, s in lay[len(W.blob_layout(g)):])
    for bad in (0, 65):
        with pytest.raises(ValueError):
            W.classifier_blob_layout(dict(g, num_labels=bad))
    assert not W.random_classifier_blob(g, 0)[-128:].any()  # zero bias, zero padding


def _hf_state(flat, g):
    return {k: v.detach().numpy().copy() for k, v in RR.build_hf_classifier(flat, g).state_dict().items()}


def test_state_dict_and_hf_dir_loading(tmp_path):
    from b200rt import weights as W

    g = R.BertGeometry(layers=2, hidden=384, heads=12, inter=1536)
    flat = RR.make_classifier_weights(g, 4, "trained", 3)
    sd = _hf_state(flat, g)
    gd, blob = W.load_hf_classifier_state_dict(sd, W.geometry_from_state_dict(sd, 1e-12, 12))
    assert gd["num_labels"] == 3 and gd["layers"] == 2 and gd["heads"] == 12
    assert np.array_equal(blob.view(np.uint32), RR.pack_classifier_blob(flat, g).view(np.uint32))
    # a snapshot directory: config.json names the architecture and the labels
    W.write_safetensors(str(tmp_path / "model.safetensors"), {k: v.astype(np.float32) for k, v in sd.items() if v.dtype.kind == "f"})
    cfg = {"architectures": ["BertForSequenceClassification"], "num_attention_heads": 12, "layer_norm_eps": 1e-12,
           "id2label": {"0": "neg", "1": "neu", "2": "pos"}}
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    gd2, blob2 = W.load_hf_dir(str(tmp_path))
    assert gd2["id2label"] == {0: "neg", 1: "neu", 2: "pos"} and gd2["num_labels"] == 3
    assert np.array_equal(blob2.view(np.uint32), blob.view(np.uint32))
    cfg.pop("id2label")
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    assert W.load_hf_dir(str(tmp_path))[0]["id2label"] == {0: "LABEL_0", 1: "LABEL_1", 2: "LABEL_2"}
    # the same snapshot without the architecture loads as the encoder alone (an embedding model)
    cfg.pop("architectures")
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    ge, be = W.load_hf_dir(str(tmp_path))
    assert "num_labels" not in ge and be.size == W.blob_numel(ge)


def test_loader_refusals():
    from b200rt import weights as W

    g = R.BertGeometry(layers=1, hidden=384, heads=12, inter=1536)
    sd = _hf_state(RR.make_classifier_weights(g, 1, "hf", 1), g)
    no_pool = {k: v for k, v in sd.items() if "pooler" not in k}
    with pytest.raises(ValueError, match="add_pooling_layer=False"):
        W.load_hf_classifier_state_dict(no_pool, W.geometry_from_state_dict(no_pool, 1e-12, 12))
    no_cls = {k: v for k, v in sd.items() if not k.startswith("classifier.")}
    with pytest.raises(KeyError):
        W.load_hf_classifier_state_dict(no_cls, W.geometry_from_state_dict(no_cls, 1e-12, 12))


def test_abi_classifier_config_layout():
    """b200rt_bert_classifier_config: b200rt_bert_config unchanged, num_labels after it."""
    import b200rt

    assert ctypes.sizeof(b200rt.BertConfig) == 32
    assert ctypes.sizeof(b200rt.BertClassifierConfig) == 36 and b200rt.BertClassifierConfig.num_labels.offset == 32
    hdr = open(os.path.join(ROOT, "include", "b200rt.h")).read()
    assert "b200rt_bert_config bert;\n    int32_t num_labels;" in hdr


# ================================================================================================ router scoring

def test_router_scoring():
    from tei_router import server as S

    z = np.array([[2.0], [-1.0], [0.5], [2.0]])
    s = S.label_scores(z, False)[:, 0]
    assert np.allclose(s, 1.0 / (1.0 + np.exp(-z[:, 0])))
    r = S.rerank_response(z, ["a", "b", "c", "d"], raw_scores=False, return_text=True)
    assert [x["index"] for x in r] == [0, 3, 2, 1] and r[0]["text"] == "a" and abs(r[2]["score"] - s[2]) < 1e-15
    r = S.rerank_response(z, ["a", "b", "c", "d"], raw_scores=True, return_text=False)
    assert [x["score"] for x in r] == [2.0, 2.0, 0.5, -1.0] and "text" not in r[0]
    big = S.label_scores(np.array([[-800.0], [800.0]]), False)[:, 0]  # no overflow warnings, exact saturation
    assert big[0] == 0.0 and big[1] == 1.0
    # /predict: softmax over labels, sorted, id2label names
    row = np.array([0.1, 2.0, -1.0])
    p = S.predict_response(row, {0: "neg", 1: "neu", 2: "pos"}, False)
    e = np.exp(row - row.max())
    assert [x["label"] for x in p] == ["neu", "neg", "pos"] and abs(p[0]["score"] - e[1] / e.sum()) < 1e-15
    assert [x["score"] for x in S.predict_response(row, {}, True)] == [2.0, 0.1, -1.0]
    assert [x["label"] for x in S.predict_response(row, {}, True)] == ["LABEL_1", "LABEL_0", "LABEL_2"]
    assert S.predict_response(np.array([0.0]), {0: "LABEL_0"}, False) == [{"label": "LABEL_0", "score": 0.5}]
    assert S.parse_predict_inputs("x") == (["x"], False)
    assert S.parse_predict_inputs(["q", "p"]) == ([("q", "p")], False)
    assert S.parse_predict_inputs(["a", "b", "c"]) == (["a", "b", "c"], True)
    assert S.parse_predict_inputs([["q", "p"], "s"]) == ([("q", "p"), "s"], True)
    for bad in ([], 3, [["a"]], [1, 2, 3]):
        with pytest.raises(TypeError):
            S.parse_predict_inputs(bad)


def test_router_model_table():
    from tei_router import server as S

    g = S.geometry_for_model_id("cross-encoder/ms-marco-MiniLM-L-6-v2")
    assert g["num_labels"] == 1 and g["layers"] == 6 and g["hidden"] == 384 and g["heads"] == 12
    assert S.geometry_for_model_id("cross-encoder/ms-marco-MiniLM-L-12-v2")["layers"] == 12
    assert "num_labels" not in S.geometry_for_model_id("BAAI/bge-base-en-v1.5")


# ================================================================================================ kernel references

def _embed_case(W=384, B=4, S=64, seed=0):
    rng = np.random.default_rng(seed)
    vocab = 500
    word = rng.standard_normal((vocab, W), dtype=np.float32) * np.float32(0.5)
    pos = rng.standard_normal((S, W), dtype=np.float32) * np.float32(0.5)
    type2 = rng.standard_normal((2, W), dtype=np.float32) * np.float32(0.5)
    ids = rng.integers(0, vocab, size=B * S).astype(np.int32)
    segs = np.array([1, 30, S, 63][:B], np.int32)
    return ids, segs, word, pos, type2, S


def test_check_embed_segs_accepts_emulation_rejects_mutants():
    args = _embed_case()
    hi, lo, st = RR.emulate_embed_segs(*args)
    RR.check_embed_segs("emulated embed segs", hi, lo, st, *args)
    for mutant in RR.EMBED_MUTANTS:
        hi, lo, st = RR.emulate_embed_segs(*args, mutant=mutant)
        with pytest.raises(AssertionError):
            RR.check_embed_segs(f"mutant {mutant}", hi, lo, st, *args)
    # segs outside [0, S] clamp: -5 is 0 (all type 1), S + 9 is S (all type 0)
    ids, _, word, pos, type2, S = args
    segs = np.array([-5, S + 9, 0, S], np.int32)
    a = RR.embed_segs_exact(ids, segs, word, pos, type2, S)[2]
    b = RR.embed_segs_exact(ids, np.array([0, S, 0, S]), word, pos, type2, S)[2]
    assert np.array_equal(a, b)


def _head_case(W=384, L=2, B=5, S=3, seed=0):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((B * S, W)) * 2.0 + rng.standard_normal(W) * 0.5).astype(np.float32)
    hi, lo = KR.split_hilo(x)
    gamma = (1.0 + 0.1 * rng.standard_normal(W)).astype(np.float32)
    beta = (0.05 * rng.standard_normal(W)).astype(np.float32)
    pw = (rng.standard_normal((W, W)) * 1.5 / np.sqrt(W)).astype(np.float32)
    pb = (0.1 * rng.standard_normal(W)).astype(np.float32)
    cw = (rng.standard_normal((L, W)) * 0.3).astype(np.float32)
    cb = np.zeros(128, np.float32)
    cb[:L] = rng.standard_normal(L)
    return hi, lo, gamma, beta, pw, pb, cw, cb, S, 1e-12


@pytest.mark.parametrize("W,L", [(384, 1), (768, 2), (1024, 64)])
def test_check_cls_head_accepts_emulation_rejects_mutants(W, L):
    args = _head_case(W, L)
    RR.check_cls_head(f"emulated cls_head W={W} L={L}", RR.emulate_cls_head(*args), *args)
    for mutant in RR.HEAD_MUTANTS:
        if mutant == "wc_transposed" and L == 1:
            continue  # a [1, W] matrix reads the same either way
        with pytest.raises(AssertionError):
            RR.check_cls_head(f"mutant {mutant}", RR.emulate_cls_head(*args, mutant=mutant), *args)
