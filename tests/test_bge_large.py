"""CPU: the bge-large geometry (hidden 1024, 16 heads of 64, inter 4096) off the GPU -- the oracle against the HF golden vectors,
the weight loader's head count, the router's geometry table, the blob size, the per-model wave capacity -- and the kernel-level
checks of tests/test_gpu_bge_large.py shown to discriminate: a numpy emulation of the 16-head attention and of the 8-partial row
statistics passes them, and each mutant standing for a plausible rewrite bug fails them (a 12-head unit decode over a 16-head
layout, K / V read at bge-base's 12 * 64 column offset, six or seven partials read where there are eight, the last partial
dropped, a 99-item capacity computed as 132)."""
import importlib.util
import json
import os

import numpy as np
import pytest

import attention_refs as AR
import kernel_refs as KR
import mean_pool_refs as MP
from oracle import bge_ref as R
from b200rt import weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_large_golden", os.path.join(ROOT, "tests", "golden", "make_large_golden.py"))
mlg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mlg)

HD, NH, H = 64, 16, 1024


# ================================================================================================ oracle, weights, router

@pytest.fixture(scope="module")
def large_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "bge_large_golden.npz"))


_weights = {}


def _flat(layers, style, seed):
    key = (layers, style, seed)
    if key not in _weights:
        _weights.clear()  # one 24-layer model in memory at a time
        _weights[key] = R.make_weights(mlg.geometry(layers), seed, style)
    return _weights[key]


@pytest.mark.parametrize("case", sorted(mlg.CASES, key=lambda c: mlg.CASES[c][:3]))
def test_oracle_matches_large_golden(large_golden, case):
    layers, style, wseed, spec, pooling = mlg.CASES[case]
    g = mlg.geometry(layers)
    assert (g.hidden, g.heads, g.head_dim, g.inter) == (1024, 16, 64, 4096)
    flat = _flat(layers, style, wseed)
    ids, lens = mlg.case_inputs(spec)
    assert np.array_equal(np.frombuffer(bytes.fromhex(mlg.blob_digest(flat, g)), np.uint8), large_golden[f"{case}_digest"])
    assert int(ids.astype(np.int64).sum()) == int(large_golden[f"{case}_ids_sum"][0])
    fwd = MP.forward_np_mean if pooling == "mean" else R.forward_np
    rel = R.rel_l2(fwd(flat, ids, lens, g), large_golden[f"{case}_emb"])
    print(f"case {case}: oracle vs HF fp32 golden {rel.max():.3e}")
    assert rel.max() <= 5e-6


def test_flops_per_item():
    assert round(mlg.geometry(24).flops_per_item(512) / 1e9, 1) == 335.0


def _snapshot(tmp_path, g, seed, config):
    flat = R.make_weights(g, seed, "trained")
    snap = tmp_path / "models--BAAI--bge-large-en-v1.5" / "snapshots" / "rev0"
    snap.mkdir(parents=True)
    W.write_safetensors(str(snap / "model.safetensors"), {k: np.ascontiguousarray(v) for k, v in R.flat_to_hf_state(flat, g).items()})
    if config is not None:
        (snap / "config.json").write_text(json.dumps(config))
    return flat, snap


@pytest.mark.parametrize("with_heads", [True, False])
def test_weights_round_trip_with_sixteen_heads(tmp_path, with_heads):
    """With num_attention_heads in config.json, and without it: the hidden // 64 fallback is right (16) for hidden 1024."""
    g = R.BertGeometry(vocab=97, hidden=1024, layers=2, heads=16, inter=4096, max_pos=40)
    cfg = {"hidden_size": 1024, "layer_norm_eps": 1e-12}
    if with_heads:
        cfg["num_attention_heads"] = 16
    flat, snap = _snapshot(tmp_path, g, 4, cfg)
    assert W.resolve_hub_snapshot(str(tmp_path), "BAAI/bge-large-en-v1.5") == str(snap)
    geo, blob = W.load_hf_dir(str(snap))
    assert geo == R.geometry_dict(g) and geo["heads"] == 16
    assert np.array_equal(blob, R.pack_blob(flat, g))
    assert W.BGE_LARGE_GEOMETRY == R.geometry_dict(mlg.geometry(24))


def test_router_geometry_per_model_id():
    from tei_router import server

    assert server.geometry_for_model_id("BAAI/bge-large-en-v1.5") == W.BGE_LARGE_GEOMETRY
    assert server.geometry_for_model_id("BAAI/bge-small-en-v1.5") == W.BGE_SMALL_GEOMETRY
    assert server.geometry_for_model_id("BAAI/bge-base-en-v1.5") == W.BGE_BASE_GEOMETRY
    assert server.geometry_for_model_id("intfloat/e5-large-v2") == W.BGE_BASE_GEOMETRY  # no table entry: geometry from config.json
    assert server.resolve_pooling(None, None, "BAAI/bge-large-en-v1.5") == "cls"


def test_blob_size_for_the_large_geometry():
    g = W.BGE_LARGE_GEOMETRY
    layout = W.blob_layout(g)
    assert W.blob_numel(g) == sum(int(np.prod(s)) for _, s in layout)
    emb = (30522 + 512 + 2) * 1024 + 2 * 1024
    per_layer = 4 * 1024 * 1024 + 2 * 1024 * 4096 + 3 * 1024 + 1024 + 2 * 1024 + 4096 + 1024 + 2 * 1024
    assert W.blob_numel(g) == emb + 24 * per_layer == 334_092_288
    assert W.blob_numel(g) == R.pack_blob(R.make_weights(mlg.geometry(1), 0, "hf"), mlg.geometry(1)).size + 23 * per_layer


# ================================================================================================ wave capacity

def _fits(rows, hidden, inter, rt_rows):
    """Every workspace buffer (sized for bge-base at rt_rows rows) holds `rows` rows of this geometry."""
    return (rows * hidden <= rt_rows * 768 and rows * 3 * hidden <= rt_rows * 2304 and rows * inter <= rt_rows * 3072
            and rows * (hidden // 128) <= rt_rows * 6)


def spec_cap_rows(hidden, rt_rows):
    """The per-model row capacity the engine must compute (engine.cu model_cap_rows; the GPU suite compares the engine's value,
    b200rt_debug_model_cap_rows, with this): min(R, R * 768 / hidden) rounded down to a multiple of 128."""
    r = rt_rows * 768 // hidden
    return rt_rows if r >= rt_rows else r // 128 * 128


def check_capacity(cap_rows):
    """What a per-model capacity function cap_rows(hidden, rt_rows) must satisfy: bge-base and bge-small keep the runtime's rows;
    bge-large's rows are whole 128-row tiles, fit every buffer and leave less than one tile unused; a 132-item runtime gives
    99 bge-large items, with bge-base's per-SM work counts in whole 2-CTA cluster pairs."""
    for items in list(range(1, 300)) + [1024]:
        R0 = items * 512
        assert cap_rows(768, R0) == cap_rows(384, R0) == R0, items
        rows = cap_rows(1024, R0)
        assert rows % 128 == 0 and _fits(rows, 1024, 4096, R0) and not _fits(rows + 128, 1024, 4096, R0), items
    assert cap_rows(1024, 132 * 512) // 512 == 99
    assert cap_rows(1024, 512) == 384  # below one item: model_load refuses the model
    # a full wave has bge-base's per-SM work counts: 396 m-tiles x 12 / 4 / 16 / 4 n-tiles, 99 x 16 attention units
    m_tiles = cap_rows(1024, 132 * 512) // 128
    assert (m_tiles * 12, m_tiles * 4, m_tiles * 16, m_tiles * 4, 99 * 16) == (528 * 9, 528 * 3, 528 * 12, 528 * 3, 132 * 12)
    assert m_tiles % 2 == 0  # whole 2-CTA cluster pairs


def test_model_capacity_is_three_quarters_for_bge_large():
    check_capacity(spec_cap_rows)


@pytest.mark.parametrize("mutant", [lambda h, r: r, lambda h, r: r * 768 // h, lambda h, r: r * 768 // h // 512 * 512],
                         ids=["bge_base_capacity_132_items", "not_tile_aligned", "rounded_to_whole_items"])
def test_capacity_mutants_fail(mutant):
    """A bge-large capacity left at bge-base's 132 items overruns the workspace; one not rounded to 128-row tiles breaks the
    tile walk; one rounded to whole items wastes rows and breaks the 99-item wave's work counts."""
    with pytest.raises(AssertionError):
        check_capacity(mutant)


# ================================================================================================ emulations and mutants

def _attention_emulated(qkv16, lens, B, S, heads=NH, head_dim=HD, decode_heads=None, kv_cols=None):
    """attention_sm90.cu's rounding in numpy: S in fp32 from fp16 operands, online softmax over 64-key sub-blocks in base 2
    with P rounded to fp16, O / l rounded to fp16.  The keywords inject rewrite bugs: `decode_heads` (the head count the unit
    decode divides by; units are still B * heads), `kv_cols` (the column offset of the K block, V at twice it)."""
    hid = heads * head_dim
    dh = decode_heads or heads
    kv = kv_cols or hid
    k2 = np.float32(1.0 / np.sqrt(head_dim) * 1.4426950408889634)
    x = np.asarray(qkv16, np.float16).astype(np.float32).reshape(B, S, 3 * hid)
    ctx = np.zeros((B, S, hid), np.float16)
    for u in range(B * heads):
        b, h = u // dh, u % dh
        if b >= B:
            continue
        n = int(np.clip(lens[b], 1, S))
        c0 = h * head_dim
        q = x[b, :, c0:c0 + head_dim]
        k = x[b, :, kv + c0:kv + c0 + head_dim]
        v = x[b, :, 2 * kv + c0:2 * kv + c0 + head_dim]
        m = np.full((S, 1), -np.inf, np.float32)
        l = np.zeros((S, 1), np.float32)
        o = np.zeros((S, head_dim), np.float32)
        for k0 in range(0, n, 64):
            s = q @ k[k0:k0 + 64].T
            s[:, max(0, n - k0):] = -np.inf
            m_new = np.maximum(m, s.max(-1, keepdims=True))
            alpha = np.exp2((m - m_new) * k2)
            p = np.exp2(s * k2 - m_new * k2).astype(np.float32)
            l = l * alpha + p.sum(-1, keepdims=True, dtype=np.float32)
            o = o * alpha + p.astype(np.float16).astype(np.float32) @ v[k0:k0 + 64]
            m = m_new
        ctx[b, :, c0:c0 + head_dim] = (o / l).astype(np.float16)
    return ctx.reshape(B * S, hid)


@pytest.fixture(scope="module")
def attn_case():
    B, S, lens = 2, 160, [160, 65]
    rng = np.random.default_rng(3)
    return (rng.standard_normal((B * S, 3 * H)) * 2.0).astype(np.float16), lens, B, S


def test_attention_emulation_passes(attn_case):
    qkv, lens, B, S = attn_case
    AR.check_attention("emulated 16-head attention", _attention_emulated(qkv, lens, B, S), qkv, lens, B, S, heads=NH, head_dim=HD)


@pytest.mark.parametrize("bug", [dict(decode_heads=12), dict(kv_cols=12 * 64)], ids=["decode_12_heads", "kv_offset_12x64"])
def test_attention_mutants_fail(attn_case, bug):
    qkv, lens, B, S = attn_case
    got = _attention_emulated(qkv, lens, B, S, **bug)
    with pytest.raises(AssertionError):
        AR.check_attention(f"mutant {bug}", got, qkv, lens, B, S, heads=NH, head_dim=HD)


def _row_stats32(p, eps, parts_read=8, width_parts=None):
    """gemm_sm90.cu row_stats<8> in fp32 over the first `parts_read` partials of each row, the row taken as 128 width_parts
    columns wide (default parts_read).  parts_read 6 / 7 with the width following is an instantiation that reads too few
    partials; parts_read 7 with width_parts 8 drops the last partial."""
    p = np.asarray(p, np.float32)[:, :parts_read]
    s, m2 = p[..., 0], p[..., 1]
    n = np.float32(128.0 * (width_parts or parts_read))
    mean = s.sum(-1, dtype=np.float32) * (np.float32(1.0) / n)
    d = s * np.float32(1.0 / 128.0) - mean[:, None]
    var = (np.float32(128.0) * d * d + m2).sum(-1, dtype=np.float32) * (np.float32(1.0) / n)
    return mean, (np.float32(1.0) / np.sqrt(var + np.float32(eps))).astype(np.float32)


@pytest.fixture(scope="module")
def stats_case():
    rng = np.random.default_rng(2)
    y = (rng.standard_normal((64, H)) * 1.7 + 0.3).astype(np.float32)
    y += np.repeat(rng.standard_normal(H // 64) * 0.5, 64)[None, :].astype(np.float32)
    y[:, 896:] += 2.0  # the last 128 columns sit apart, as a real row's outlier channels can
    p = KR.partials(y).astype(np.float32)
    assert p.shape == (64, 8, 2)
    return p, KR.stats_from_partials(p, 1e-12)


def test_row_stats_eight_partials(stats_case):
    p, (mean, rstd, mean_tol, rstd_rel) = stats_case
    m32, r32 = _row_stats32(p, 1e-12)
    KR.check("row_stats<8> mean", m32, mean, mean_tol)
    KR.check("row_stats<8> rstd", r32, rstd, rstd_rel * rstd)


@pytest.mark.parametrize("bug", [dict(parts_read=6), dict(parts_read=7), dict(parts_read=7, width_parts=8)],
                         ids=["six_partials", "seven_partials", "last_partial_dropped"])
def test_row_stats_mutants_fail(stats_case, bug):
    p, (mean, rstd, mean_tol, rstd_rel) = stats_case
    m, r = _row_stats32(p, 1e-12, **bug)
    with pytest.raises(AssertionError):
        KR.check(f"row_stats mutant {bug} mean", m, mean, mean_tol)
        KR.check(f"row_stats mutant {bug} rstd", r, rstd, rstd_rel * rstd)
