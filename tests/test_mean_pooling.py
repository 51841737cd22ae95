"""CPU: mean pooling (sentence-transformers Pooling(mean) + Normalize) -- the oracle against the MiniLM-L6 golden, the kernel's
fp64 reference and the emulation that shows it discriminates, the snapshot's Pooling config, the router's pooling resolution
and the C ABI entry points."""
import json
import os
import re

import numpy as np
import pytest

import kernel_refs as KR
import mean_pool_refs as MP
from oracle import bge_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

import importlib.util  # noqa: E402

_spec = importlib.util.spec_from_file_location("make_minilm_golden", os.path.join(GOLDEN, "make_minilm_golden.py"))
mmg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mmg)


@pytest.fixture(scope="module")
def minilm_golden():
    return np.load(os.path.join(GOLDEN, "minilm_golden.npz"))


_weights = {}


def _flat(style, seed):
    if (style, seed) not in _weights:
        _weights[(style, seed)] = R.make_weights(mmg.geometry(), seed, style)
    return _weights[(style, seed)]


# ================================================================================================ oracle vs golden

@pytest.mark.parametrize("case", list(mmg.CASES))
def test_numpy_oracle_matches_the_minilm_golden(minilm_golden, case):
    style, seed, spec = mmg.CASES[case]
    flat = _flat(style, seed)
    ids, lens = mmg.case_inputs(spec)
    assert bytes(minilm_golden[f"{case}_digest"]).hex() == mmg.blob_digest(flat, mmg.geometry())
    assert int(minilm_golden[f"{case}_ids_sum"][0]) == int(ids.astype(np.int64).sum())
    emb = MP.forward_np_mean(flat, ids, lens, mmg.geometry())
    rel = R.rel_l2(emb, minilm_golden[f"{case}_emb"])
    print(f"case {case}: numpy fp64 mean pooling vs HF fp32 golden {rel.max():.3e}")
    assert rel.max() <= 5e-6, rel
    assert np.allclose(np.linalg.norm(emb, axis=1), 1.0, atol=1e-6)


def test_hf_oracle_matches_the_minilm_golden(minilm_golden):
    import torch

    torch.set_num_threads(min(16, os.cpu_count() or 4))
    g = mmg.geometry()
    for case in ("B", "C"):
        style, seed, spec = mmg.CASES[case]
        ids, lens = mmg.case_inputs(spec)
        emb = MP.forward_hf_mean(R.build_hf_model(_flat(style, seed), g), ids, lens)
        assert R.rel_l2(emb, minilm_golden[f"{case}_emb"]).max() <= 5e-6


def test_golden_holds_one_token_items_and_mean_differs_from_cls(minilm_golden):
    """One-token items pool to their [CLS] row; longer items do not."""
    style, seed, spec = mmg.CASES["B"]
    ids, lens = mmg.case_inputs(spec)
    assert (lens == 1).sum() >= 2
    cls = R.forward_np(_flat(style, seed), ids, lens, mmg.geometry())
    rel = R.rel_l2(minilm_golden["B_emb"], cls)
    assert rel[lens == 1].max() <= 5e-6
    assert rel[lens > 1].min() > 1e-2


# ================================================================================================ kernel reference

def _rows(rng, n_items, S, W, garbage=True):
    """hi / lo of n_items * S rows of a trained-like residual stream (non-zero mean, a few large channels); padding rows get
    finite garbage (the caller decides which rows are padding)."""
    x = rng.standard_normal((n_items * S, W)).astype(np.float32) * 2.0 + 0.3
    x[:, :3] *= 20.0
    hi, lo = KR.split_hilo(x)
    return hi, lo


def _ln(rng, W):
    return (1.0 + 0.2 * rng.standard_normal(W)).astype(np.float32), (0.1 * rng.standard_normal(W)).astype(np.float32)


def _poison_padding(hi, lo, lens, S, rng):
    """Rows past each length: +-60000 and large finite values (what a padded row may hold in a normal run)."""
    hi, lo = hi.copy(), lo.copy()
    W = hi.shape[1]
    for i, n in enumerate(lens):
        k = S - int(n)
        if k > 0:
            hi[i * S + int(n):(i + 1) * S] = (rng.choice([-60000.0, 60000.0, 3000.0], size=(k, W))).astype(np.float16)
    return hi, lo


LENS = [1, 2, 7, 63, 64, 65, 127, 128, 100, 9]


@pytest.mark.parametrize("W", [384, 768])
def test_emulated_kernel_passes_the_reference(W):
    rng = np.random.default_rng(W)
    S = 128
    hi, lo = _rows(rng, len(LENS), S, W)
    hi, lo = _poison_padding(hi, lo, LENS, S, rng)
    g, b = _ln(rng, W)
    out = MP.emulate_mean_pool(hi, lo, g, b, LENS, S, 1e-12)
    margin = MP.check_mean_pool_normalize(f"emulated mean pool W={W}", out, hi, lo, g, b, LENS, S, 1e-12)
    assert margin < 0.5  # the emulation sits well inside: the tolerance is not loose by accident of one term
    # out-of-range lengths are clamped, as the kernel clamps them
    lens_bad = [0, -3, S + 1, 10 ** 6] + LENS[4:]
    out_c = MP.emulate_mean_pool(hi, lo, g, b, lens_bad, S, 1e-12)
    MP.check_mean_pool_normalize("clamped lengths", out_c, hi, lo, g, b, lens_bad, S, 1e-12)
    assert np.array_equal(out_c[:2], MP.emulate_mean_pool(hi[:2 * S], lo[:2 * S], g, b, [1, 1], S, 1e-12))


@pytest.mark.parametrize("mutant", list(MP.MUTANTS) + ["ln1"])
@pytest.mark.parametrize("W", [384, 768])
def test_reference_rejects_every_mutant(W, mutant):
    rng = np.random.default_rng(W + 1)
    S = 128
    lens = [n for n in LENS if n < S]  # a padding row exists for every item
    hi, lo = _rows(rng, len(lens), S, W)
    hi, lo = _poison_padding(hi, lo, lens, S, rng)
    g, b = _ln(rng, W)
    if mutant == "ln1":  # the last layer's LN1 instead of its LN2
        g1, b1 = _ln(rng, W)
        out = MP.emulate_mean_pool(hi, lo, g1, b1, lens, S, 1e-12)
    else:
        out = MP.emulate_mean_pool(hi, lo, g, b, lens, S, 1e-12, mutant=mutant)
    with pytest.raises(AssertionError):
        MP.check_mean_pool_normalize(f"mutant {mutant}", out, hi, lo, g, b, lens, S, 1e-12)


@pytest.mark.parametrize("W", [384, 768])
def test_dividing_by_S_is_an_equivalent_mutant(W):
    """sum / S instead of sum / len scales each item by len / S, and Normalize removes the scale: the output cannot show it,
    so the check passes it (and a kernel that did it would still be right)."""
    rng = np.random.default_rng(W + 2)
    S = 128
    hi, lo = _rows(rng, len(LENS), S, W)
    hi, lo = _poison_padding(hi, lo, LENS, S, rng)
    g, b = _ln(rng, W)
    for m in MP.EQUIVALENT_MUTANTS:
        out = MP.emulate_mean_pool(hi, lo, g, b, LENS, S, 1e-12, mutant=m)
        MP.check_mean_pool_normalize(f"equivalent mutant {m}", out, hi, lo, g, b, LENS, S, 1e-12)


def test_tolerance_terms_are_named():
    """The bound grows with the rows one warp adds and carries the LayerNorm bound of every row."""
    assert MP.row_sum_ulps(1) == 1 and MP.row_sum_ulps(8) == 1 and MP.row_sum_ulps(9) == 2 and MP.row_sum_ulps(512) == 64
    rng = np.random.default_rng(3)
    hi, lo = _rows(rng, 2, 64, 384)
    g, b = _ln(rng, 384)
    _, t1 = MP.mean_pool_normalize_ref(hi, lo, g, b, [64, 64], 64, 1e-12)
    _, t8 = MP.mean_pool_normalize_ref(hi, lo, g, b, [8, 8], 64, 1e-12)
    assert np.all(t1 > 0) and np.all(t8 > 0)


# ================================================================================================ snapshot Pooling config

def _snapshot(tmp_path, pooling_cfg, modules=True, name="snap"):
    d = tmp_path / name
    d.mkdir()
    if modules:
        (d / "modules.json").write_text(json.dumps([
            {"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
            {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
            {"idx": 2, "name": "2", "path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}]))
    if pooling_cfg is not None:
        (d / "1_Pooling").mkdir()
        cfg = {"word_embedding_dimension": 384, "pooling_mode_cls_token": False, "pooling_mode_mean_tokens": False,
               "pooling_mode_max_tokens": False, "pooling_mode_mean_sqrt_len_tokens": False,
               "pooling_mode_weightedmean_tokens": False, "pooling_mode_lasttoken": False}
        cfg.update(pooling_cfg)
        (d / "1_Pooling" / "config.json").write_text(json.dumps(cfg))
    return str(d)


def test_pooling_from_dir(tmp_path):
    from b200rt.weights import pooling_from_dir

    assert pooling_from_dir(_snapshot(tmp_path, {"pooling_mode_cls_token": True}, name="cls")) == "cls"
    assert pooling_from_dir(_snapshot(tmp_path, {"pooling_mode_mean_tokens": True}, name="mean")) == "mean"
    assert pooling_from_dir(_snapshot(tmp_path, None, modules=False, name="plain")) is None  # a plain HF checkpoint
    assert pooling_from_dir(_snapshot(tmp_path, None, name="nocfg")) is None                # modules.json, no Pooling config
    for bad in ({"pooling_mode_max_tokens": True}, {"pooling_mode_mean_sqrt_len_tokens": True},
                {"pooling_mode_weightedmean_tokens": True}, {"pooling_mode_lasttoken": True},
                {"pooling_mode_cls_token": True, "pooling_mode_mean_tokens": True}, {}):
        d = _snapshot(tmp_path, bad, name="bad" + str(abs(hash(json.dumps(bad, sort_keys=True)))))
        with pytest.raises(ValueError, match=r"cls.*mean"):
            pooling_from_dir(d)


def test_minilm_geometry():
    from b200rt.weights import BGE_SMALL_GEOMETRY, MINILM_L6_GEOMETRY

    assert MINILM_L6_GEOMETRY == dict(BGE_SMALL_GEOMETRY, layers=6)
    assert MINILM_L6_GEOMETRY == dict(vocab=30522, hidden=384, layers=6, heads=12, inter=1536, max_pos=512, type_vocab=2, eps=1e-12)


# ================================================================================================ router

def test_router_pooling_resolution(tmp_path):
    from tei_router import server

    mean_dir = _snapshot(tmp_path, {"pooling_mode_mean_tokens": True}, name="mean")
    cls_dir = _snapshot(tmp_path, {"pooling_mode_cls_token": True}, name="cls")
    plain = _snapshot(tmp_path, None, modules=False, name="plain")
    max_dir = _snapshot(tmp_path, {"pooling_mode_max_tokens": True}, name="max")
    minilm, bge = "sentence-transformers/all-MiniLM-L6-v2", "BAAI/bge-base-en-v1.5"
    table = [
        # (--pooling, snapshot dir, model id) -> pooling
        ((None, None, bge), "cls"),              # nothing declared: cls, as before
        ((None, plain, bge), "cls"),
        ((None, None, minilm), "mean"),          # the model-id table
        ((None, plain, minilm), "mean"),
        ((None, mean_dir, bge), "mean"),         # the snapshot's Pooling config beats the table ...
        ((None, cls_dir, minilm), "cls"),
        (("cls", mean_dir, minilm), "cls"),      # ... and the flag beats both
        (("mean", cls_dir, bge), "mean"),
        (("cls", None, bge), "cls"),
        (("cls", max_dir, bge), "cls"),          # an explicit flag does not read the snapshot's config
    ]
    for args, want in table:
        assert server.resolve_pooling(*args) == want, args
    for flag in ("splade", "last-token", "max", "CLS"):
        with pytest.raises(ValueError, match="cls, mean"):
            server.resolve_pooling(flag, None, bge)
    with pytest.raises(ValueError):
        server.resolve_pooling(None, max_dir, bge)


def test_router_knows_minilm():
    from b200rt.weights import MINILM_L6_GEOMETRY
    from tei_router import server

    assert server.geometry_for_model_id("sentence-transformers/all-MiniLM-L6-v2") == MINILM_L6_GEOMETRY
    assert server.parse_args(["--model-id", "x"]).pooling is None  # unset: resolved from the snapshot / table
    assert server.parse_args(["--pooling", "mean"]).pooling == "mean"


def test_router_refuses_unsupported_pooling_before_starting(capsys):
    from tei_router import server

    assert server.main(["--pooling", "splade", "--port", "1"]) != 0
    assert "splade" in capsys.readouterr().err


def test_embed_model_rejects_unknown_pooling_before_loading():
    import b200rt

    with pytest.raises(b200rt.B200RTError) as e:
        b200rt.EmbedModel(dict(vocab=1, hidden=384, layers=1, heads=12, inter=1536, max_pos=8, type_vocab=1, eps=1e-12),
                          np.zeros(1, np.float32), pooling="max")
    assert e.value.code == b200rt.E_INVALID and "mean" in str(e.value)


# ================================================================================================ C ABI

def _declared(header):
    txt = open(os.path.join(ROOT, "include", header)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return set(re.findall(r"\b(b200rt_[a-z_0-9]+)\s*\(", txt)), txt


def test_abi_declares_and_exports_the_mean_pool_entry_points():
    import b200rt

    lib = b200rt.load_library()
    decl, txt = _declared("b200rt.h")
    decl_dbg, _ = _declared("b200rt_debug.h")
    assert "b200rt_model_load_ex" in decl and "b200rt_model_load_ex" in b200rt.ABI_SYMBOLS
    assert "b200rt_debug_mean_pool_normalize" in decl_dbg and "b200rt_debug_mean_pool_normalize" in b200rt.DEBUG_SYMBOLS
    assert re.search(r"#define\s+B200RT_LOAD_POOL_MEAN\s+1u\b", txt)
    assert b200rt.LOAD_POOL_MEAN == 1
    for name in ("b200rt_model_load_ex", "b200rt_debug_mean_pool_normalize", "b200rt_model_load"):
        assert hasattr(lib, name), name
