"""CPU: SPLADE sparse encoders -- the fp64 oracle against HF BertForMaskedLM, the `splade` weight style's statistics, the
masked-LM loaders and blob layout, the router's --pooling splade resolution and /embed_sparse formatting, and that the
kernel checks of tests/test_gpu_splade.py accept an emulation of each SPLADE launch and reject its mutants."""
import json
import os

import numpy as np
import pytest

import kernel_refs as KR
import splade_refs as SR
from oracle import bge_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def splade2():
    g = R.BertGeometry(layers=2)
    return g, SR.make_splade_weights(g, 5, "splade")


# ------------------------------------------------------------------------------------------------ oracle

def _golden_module():
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_splade_golden", os.path.join(ROOT, "tests", "golden", "make_splade_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_golden_is_small_and_holds_every_case():
    msg = _golden_module()
    path = os.path.join(ROOT, "tests", "golden", "splade_golden.npz")
    assert os.path.getsize(path) < 100_000
    golden = np.load(path)
    for name in msg.CASES:
        cols, v = msg.reference(golden, name)
        assert v.shape == (len(msg.LENS), len(cols)) and (v >= 0).all()
        assert (cols[-32:] == np.arange(msg.VOCAB - 32, msg.VOCAB)).all()


@pytest.mark.parametrize("name", ["base2_hf", "base2_splade", "base12_splade", "small2_splade"])
def test_oracle_matches_golden(name):
    """splade_np (fp64) against HF BertForMaskedLM fp32 as the golden recorded it, on the golden's own inputs."""
    msg = _golden_module()
    golden = np.load(os.path.join(ROOT, "tests", "golden", "splade_golden.npz"))
    ids, lens = golden["ids"], golden["lens"]
    assert np.array_equal(ids, msg.inputs()[0]) and np.array_equal(lens, msg.inputs()[1])
    cols, hf = msg.reference(golden, name)
    ref = SR.splade_np(msg.weights(name), ids, lens, msg.geometry(name))[:, cols]
    err = np.abs(hf - ref).max()
    print(f"{name}: oracle vs HF golden max |err| {err:.2e}, rel-L2 {R.rel_l2(hf, ref).max():.2e}")
    assert err < 2e-5


@pytest.mark.parametrize("style", SR.STYLES)
def test_oracle_matches_hf(style, splade2):
    """HF BertForMaskedLM (fp32, decoder tied) + SpladePooling(max, relu) against the fp64 oracle: fp32 noise."""
    g = R.BertGeometry(layers=2)
    flat = splade2[1] if style == "splade" else SR.make_splade_weights(g, 5, "hf")
    ids, lens = R.synth_ragged(3, 140, seed=3, min_len=1)
    lens[0] = 1
    ref = SR.splade_np(flat, ids, lens, g)
    hf = SR.splade_hf(SR.build_hf_masked_lm(flat, g), ids, lens)
    err = np.abs(hf - ref).max()
    print(f"{style}: HF fp32 vs fp64 oracle max |err| {err:.2e} (values up to {ref.max():.2f})")
    assert err < 2e-5 * max(1.0, ref.max())
    assert ((hf > 0) == (ref > 0))[np.abs(ref) > 1e-4].all()


def test_splade_style_statistics(splade2):
    """The `splade` style on a seeded batch of 64-256-token items keeps 50-400 non-zero words per item with values up to a few
    units, as trained SPLADE documents do; the one-token item keeps a handful."""
    g, flat = splade2
    ids, lens = R.synth_ragged(6, 256, seed=77, min_len=64)
    out = SR.splade_np(flat, ids, lens, g)
    nnz = (out > 0).sum(1)
    print(f"non-zero words {nnz.tolist()} for lengths {lens.tolist()}; max value {out.max():.2f}")
    assert (nnz >= 50).all() and (nnz <= 400).all()
    assert 1.0 < out.max() < 5.0
    one = SR.splade_np(flat, ids[:1, :1], np.array([1]), g)
    assert 0 < (one > 0).sum() < 50
    assert (flat["mlm.dec.b"] < 0).all() and np.array_equal(flat["mlm.dec.w"], flat["emb.word"])


def test_fp16_operand_floor_is_small(splade2):
    g, flat = splade2
    ids, lens = R.synth_ragged(3, 128, seed=4, min_len=60)
    ref = SR.splade_np(flat, ids, lens, g)
    fl = SR.splade_fp16_operands(flat, ids, lens, g)
    assert R.rel_l2(fl, ref).max() < 4e-3


# ------------------------------------------------------------------------------------------------ weights and loaders

def _hf_state_dict(flat, g, with_decoder=True, bias_key="cls.predictions.bias"):
    sd = {"bert." + k: v for k, v in R.flat_to_hf_state({k: v for k, v in flat.items() if not k.startswith("mlm.")}, g).items()}
    t = "cls.predictions.transform."
    sd.update({t + "dense.weight": flat["mlm.t.w"], t + "dense.bias": flat["mlm.t.b"], t + "LayerNorm.weight": flat["mlm.ln.g"],
               t + "LayerNorm.bias": flat["mlm.ln.b"], bias_key: flat["mlm.dec.b"]})
    if with_decoder:
        sd["cls.predictions.decoder.weight"] = flat["mlm.dec.w"]
    return {k: np.ascontiguousarray(v, np.float32) for k, v in sd.items()}


def test_splade_blob_layout_and_random_blob():
    from b200rt import weights as W

    g = dict(W.BGE_SMALL_GEOMETRY, layers=2)
    lay = W.splade_blob_layout(g)
    assert [n for n, _ in lay[-6:]] == ["mlm.t.w", "mlm.t.b", "mlm.ln.g", "mlm.ln.b", "mlm.dec.w", "mlm.dec.b"]
    assert lay[-1][1] == (30592,) and lay[-2][1] == (30522, 384)
    blob = W.random_splade_blob(g, 3)
    n = W.blob_numel(g)
    assert blob.size == sum(int(np.prod(s)) for _, s in lay)
    assert np.array_equal(blob[:n], W.random_blob(g, 3))


def test_masked_lm_state_dict_and_dir_loading(tmp_path, splade2):
    """HF state dict (torch tensors), safetensors with decoder.weight, and a tied safetensors checkpoint without it (decoder =
    word embeddings) all load to pack_splade_blob's bits; the bias may come as decoder.bias."""
    import torch
    from b200rt import weights as W

    g, flat = splade2
    want = SR.pack_splade_blob(flat, g)
    model = SR.build_hf_masked_lm(flat, g)
    geo, blob = W.load_hf_masked_lm_state_dict(model.state_dict())
    assert geo == R.geometry_dict(g) and np.array_equal(blob, want)
    geo, blob = W.load_hf_masked_lm_state_dict(_hf_state_dict(flat, g, bias_key="cls.predictions.decoder.bias"))
    assert np.array_equal(blob, want)
    for with_dec in (True, False):
        d = tmp_path / f"dec{int(with_dec)}"
        d.mkdir()
        W.write_safetensors(str(d / "model.safetensors"), _hf_state_dict(flat, g, with_dec))
        (d / "config.json").write_text(json.dumps({"architectures": ["BertForMaskedLM"], "layer_norm_eps": 1e-12,
                                                   "num_attention_heads": 12}))
        assert W.is_masked_lm_dir(str(d))
        geo, blob = W.load_hf_masked_lm_dir(str(d))
        assert geo == R.geometry_dict(g) and np.array_equal(blob, want), with_dec
    # a snapshot without a config.json is recognised by its head
    os.remove(tmp_path / "dec0" / "config.json")
    assert W.is_masked_lm_dir(str(tmp_path / "dec0"))
    del torch


def test_masked_lm_loader_refusals(splade2):
    from b200rt import weights as W

    g, flat = splade2
    sd = _hf_state_dict(flat, g)
    no_head = {k: v for k, v in sd.items() if not k.startswith("cls.predictions.transform.")}
    with pytest.raises(ValueError, match="BertForMaskedLM"):
        W.load_hf_masked_lm_state_dict(no_head)
    no_bias = {k: v for k, v in sd.items() if k != "cls.predictions.bias"}
    with pytest.raises(KeyError):
        W.load_hf_masked_lm_state_dict(no_bias)
    assert not W.has_masked_lm_head(no_head)


def test_abi_declares_the_splade_entries():
    import b200rt

    for name in ("b200rt_debug_gemm_splade", "b200rt_debug_mlm_ln_stats", "b200rt_debug_splade_finalize"):
        assert name in b200rt.DEBUG_SYMBOLS
        assert name in open(os.path.join(ROOT, "include", "b200rt_debug.h")).read()
    assert '"bert_splade"' in open(os.path.join(ROOT, "include", "b200rt.h")).read()


# ------------------------------------------------------------------------------------------------ router

def test_router_resolves_splade(tmp_path, splade2):
    """--pooling splade: served for a masked-LM snapshot (config or weights) and for the SPLADE ids; refused, with the
    message every other unsupported pooling gets, for bge and for a BertModel snapshot."""
    from b200rt import weights as W
    from tei_router import server

    g, flat = splade2
    mlm = tmp_path / "mlm"
    mlm.mkdir()
    W.write_safetensors(str(mlm / "model.safetensors"), _hf_state_dict(flat, g, False))
    enc = tmp_path / "enc"
    enc.mkdir()
    W.write_safetensors(str(enc / "model.safetensors"),
                        {k: np.ascontiguousarray(v) for k, v in R.flat_to_hf_state({k: v for k, v in flat.items() if not k.startswith("mlm.")}, g).items()})
    (enc / "config.json").write_text(json.dumps({"architectures": ["BertModel"]}))
    bge = "BAAI/bge-base-en-v1.5"
    assert server.resolve_pooling("splade", str(mlm), "local/x") == "splade"
    for mid in server.SPLADE_MODEL_IDS:
        assert server.resolve_pooling("splade", None, mid) == "splade"
        assert server.geometry_for_model_id(mid) == W.BGE_BASE_GEOMETRY
    for d, mid in ((None, bge), (str(enc), bge), (str(enc), "local/x")):
        with pytest.raises(ValueError, match="cls, mean"):
            server.resolve_pooling("splade", d, mid)
    assert server.resolve_pooling(None, str(mlm), bge) == "cls"  # splade only when asked for, as in TEI
    args = server.parse_args(["--model-id", "local/x", "--weights", str(enc), "--pooling", "splade"])
    with pytest.raises(ValueError, match="masked-LM"):
        server.load_splade_weights(args)
    args = server.parse_args(["--model-id", "naver/splade-v3", "--pooling", "splade"])
    geo, blob, source = server.load_splade_weights(args)
    assert source is None and np.array_equal(blob, W.random_splade_blob(geo, 0))


def test_router_sparse_response():
    from tei_router import server

    v = np.zeros((2, 10), np.float32)
    v[0, [7, 2]] = [0.5, 1.25]
    assert server.splade_response(v) == [[{"index": 2, "value": 1.25}, {"index": 7, "value": 0.5}], []]


# ------------------------------------------------------------------------------------------------ kernel checks

def _gemm_case(seed=0, B=4, S=128, K=384, vocab=600):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B * S, K))
    u = (x * (x > -0.5) * 1.3 + 0.2 * rng.standard_normal(K)).astype(np.float16)
    stats = KR.partials(u.astype(np.float64)).astype(np.float32)
    w = (rng.standard_normal((vocab, K)) / np.sqrt(K)).astype(np.float16)
    N = SR.vpad(vocab)
    c = (rng.standard_normal(N) - 1.0).astype(np.float32)
    c[rng.random(N) < 0.2] = -20.0
    lens = np.array([1, S, 63, 100], np.int32)
    return u, w, c, stats, lens, S, N, 1e-12


GEMM_MUTANTS = ("pad_row", "neighbour", "no_relu", "no_stats", "shift8", "past_vocab")


def test_check_gemm_splade_accepts_emulation_rejects_mutants():
    u, w, c, stats, lens, S, N, eps = _gemm_case()
    good = SR.emulate_gemm_splade(u, w, c, stats, lens, S, N, eps)
    SR.check_gemm_splade("emulated gemm_splade", good, u, w, c, stats, lens, S, eps)
    for mutant in GEMM_MUTANTS:
        bad = SR.emulate_gemm_splade(u, w, c, stats, lens, S, N, eps, mutant=mutant)
        with pytest.raises(AssertionError):
            SR.check_gemm_splade(f"mutant {mutant}", bad, u, w, c, stats, lens, S, eps)


def test_check_splade_finalize_rejects_logf():
    bits = SR.finalize_probe()
    SR.check_splade_finalize("emulated finalize", SR.emulate_splade_finalize(bits, 500), bits, 500)
    with pytest.raises(AssertionError):
        SR.check_splade_finalize("mutant logf", SR.emulate_splade_finalize(bits, 500, mutant="logf"), bits, 500)
