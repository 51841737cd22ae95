"""CPU: the bge-small geometry (hidden 384, 12 heads of 32, inter 1536) off the GPU -- the oracle against the HF golden
vectors, the weight loader's head count, the router's geometry table -- and the kernel-level checks of
tests/test_gpu_bge_small.py shown to discriminate: a numpy emulation of the d = 32 attention and of the 3-partial row
statistics passes them, and each mutant standing for a plausible rewrite bug fails them (scale 1/8 instead of 1/sqrt(32), a
head read at a 64-column stride, two heads swapped, six partials read where there are three, the V half of a 64-byte row
dropped)."""
import importlib.util
import json
import os

import numpy as np
import pytest

import attention_refs as AR
import kernel_refs as KR
from oracle import bge_ref as R
from b200rt import weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_small_golden", os.path.join(ROOT, "tests", "golden", "make_small_golden.py"))
msg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(msg)

HD, H = 32, 384


# ================================================================================================ oracle, weights, router

@pytest.fixture(scope="module")
def small_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "bge_small_golden.npz"))


@pytest.mark.parametrize("case", list(msg.CASES))
def test_oracle_matches_small_golden(small_golden, case):
    layers, style, wseed, spec = msg.CASES[case]
    g = msg.geometry(layers)
    assert (g.hidden, g.heads, g.head_dim, g.inter) == (384, 12, 32, 1536)
    flat = R.make_weights(g, wseed, style)
    ids, lens = msg.case_inputs(spec)
    assert np.array_equal(np.frombuffer(bytes.fromhex(msg.blob_digest(flat, g)), np.uint8), small_golden[f"{case}_digest"])
    assert int(ids.astype(np.int64).sum()) == int(small_golden[f"{case}_ids_sum"][0])
    rel = R.rel_l2(R.forward_np(flat, ids, lens, g), small_golden[f"{case}_emb"])
    print(f"case {case}: oracle vs HF fp32 golden {rel.max():.3e}")
    assert rel.max() <= 5e-6


def test_flops_per_item():
    assert round(R.BertGeometry().flops_per_item(512) / 1e9, 2) == 96.64
    assert round(msg.geometry(12).flops_per_item(512) / 1e9, 2) == 26.58


def _snapshot(tmp_path, g, seed, config):
    flat = R.make_weights(g, seed, "trained")
    snap = tmp_path / "models--BAAI--bge-small-en-v1.5" / "snapshots" / "rev0"
    snap.mkdir(parents=True)
    W.write_safetensors(str(snap / "model.safetensors"), {k: np.ascontiguousarray(v) for k, v in R.flat_to_hf_state(flat, g).items()})
    if config is not None:
        (snap / "config.json").write_text(json.dumps(config))
    return flat, snap


def test_weights_round_trip_with_twelve_heads(tmp_path):
    g = R.BertGeometry(vocab=97, hidden=384, layers=2, heads=12, inter=1536, max_pos=40)
    flat, snap = _snapshot(tmp_path, g, 4, {"hidden_size": 384, "num_attention_heads": 12, "layer_norm_eps": 1e-12})
    assert W.resolve_hub_snapshot(str(tmp_path), "BAAI/bge-small-en-v1.5") == str(snap)
    geo, blob = W.load_hf_dir(str(snap))
    assert geo == R.geometry_dict(g) and geo["heads"] == 12
    assert np.array_equal(blob, R.pack_blob(flat, g))
    assert W.BGE_SMALL_GEOMETRY == R.geometry_dict(msg.geometry(12))


def test_hidden_384_without_config_raises(tmp_path):
    g = R.BertGeometry(vocab=97, hidden=384, layers=1, heads=12, inter=1536, max_pos=40)
    _, snap = _snapshot(tmp_path, g, 4, None)
    with pytest.raises(ValueError, match="num_attention_heads"):
        W.load_hf_dir(str(snap))
    with pytest.raises(ValueError, match="num_attention_heads"):
        W.load_hf_state_dict(R.flat_to_hf_state(R.make_weights(g, 1, "hf"), g))


def test_router_geometry_per_model_id():
    from tei_router import server

    assert server.geometry_for_model_id("BAAI/bge-small-en-v1.5") == W.BGE_SMALL_GEOMETRY
    assert server.geometry_for_model_id("BAAI/bge-base-en-v1.5") == W.BGE_BASE_GEOMETRY
    assert server.geometry_for_model_id("someone/unknown-model") == W.BGE_BASE_GEOMETRY
    args = server.parse_args(["--model-id", "BAAI/bge-small-en-v1.5"])
    args.huggingface_hub_cache = None
    g, blob, source = server.load_weights(args)
    assert source is None and g["hidden"] == 384 and blob.size == W.blob_numel(W.BGE_SMALL_GEOMETRY)


# ================================================================================================ emulations and mutants

def _attention_emulated(qkv16, lens, B, S, head_dim=HD, heads=12, scale=None, stride=None, swap=None, drop_v_half=False):
    """attention_sm90.cu's rounding in numpy at head_dim: S in fp32 from fp16 operands, online softmax over 64-key sub-blocks
    in base 2 with P rounded to fp16, O / l rounded to fp16.  The keywords inject rewrite bugs: `scale` (softmax scale),
    `stride` (columns between heads), `swap` (a pair of heads whose outputs trade places), `drop_v_half` (only the first 32
    bytes of every 64-byte V row arrive)."""
    hid = heads * head_dim
    stride = stride or head_dim
    k2 = np.float32((scale if scale is not None else 1.0 / np.sqrt(head_dim)) * 1.4426950408889634)
    x = np.asarray(qkv16, np.float16).astype(np.float32).reshape(B, S, 3 * hid)
    ctx = np.zeros((B, S, hid), np.float16)
    for b in range(B):
        n = int(np.clip(lens[b], 1, S))
        for h in range(heads):
            c0 = (h * stride) % hid  # a 64-column stride runs off the Q block at head 6 and wraps
            q = x[b, :, c0:c0 + head_dim]
            k = x[b, :, hid + c0:hid + c0 + head_dim]
            v = x[b, :, 2 * hid + c0:2 * hid + c0 + head_dim].copy()
            if drop_v_half:
                v[:, head_dim // 2:] = 0.0
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
            ctx[b, :, h * head_dim:(h + 1) * head_dim] = (o / l).astype(np.float16)
        if swap is not None:
            i, j = swap
            a, c = ctx[b, :, i * head_dim:(i + 1) * head_dim].copy(), ctx[b, :, j * head_dim:(j + 1) * head_dim].copy()
            ctx[b, :, i * head_dim:(i + 1) * head_dim], ctx[b, :, j * head_dim:(j + 1) * head_dim] = c, a
    return ctx.reshape(B * S, hid)


@pytest.fixture(scope="module")
def attn_case():
    B, S, lens = 2, 160, [160, 65]
    rng = np.random.default_rng(3)
    return (rng.standard_normal((B * S, 3 * H)) * 2.0).astype(np.float16), lens, B, S


def test_attention_reference_at_d64_is_the_bge_base_reference():
    """attention_refs at head_dim 64 gives kernel_refs.attention_ref's reference and tolerance exactly."""
    B, S, lens = 2, 96, [96, 33]
    qkv = (np.random.default_rng(1).standard_normal((B * S, 2304)) * 2.0).astype(np.float16)
    ref, tol = AR.attention_ref(qkv, lens, B, S, head_dim=64)
    ref0, tol0 = KR.attention_ref(qkv, lens, B, S)
    assert np.array_equal(ref, ref0) and np.array_equal(tol, tol0)


def test_attention_emulation_passes(attn_case):
    qkv, lens, B, S = attn_case
    AR.check_attention("emulated d=32 attention", _attention_emulated(qkv, lens, B, S), qkv, lens, B, S, head_dim=HD)


@pytest.mark.parametrize("bug", [dict(scale=0.125), dict(stride=64), dict(swap=(3, 4)), dict(drop_v_half=True)],
                         ids=["scale_one_eighth", "head_stride_64", "heads_swapped", "v_half_dropped"])
def test_attention_mutants_fail(attn_case, bug):
    qkv, lens, B, S = attn_case
    got = _attention_emulated(qkv, lens, B, S, **bug)
    with pytest.raises(AssertionError):
        AR.check_attention(f"mutant {bug}", got, qkv, lens, B, S, head_dim=HD)


def _row_stats32(p, eps, parts_read=3):
    """gemm_sm90.cu row_stats<3> in fp32; parts_read = 6 is the bug of the 768-wide instantiation reading a 3-partial row
    (the next row's partials taken for the missing three, the row width taken as 768)."""
    p = np.asarray(p, np.float32)
    flat = p.reshape(-1, 2)
    rows = p.shape[0]
    idx = (np.arange(rows)[:, None] * 3 + np.arange(parts_read)[None, :]) % flat.shape[0]
    q = flat[idx]
    s, m2 = q[..., 0], q[..., 1]
    n = np.float32(128.0 * parts_read)
    mean = s.sum(-1, dtype=np.float32) * (np.float32(1.0) / n)
    d = s * np.float32(1.0 / 128.0) - mean[:, None]
    var = (np.float32(128.0) * d * d + m2).sum(-1, dtype=np.float32) * (np.float32(1.0) / n)
    return mean, (np.float32(1.0) / np.sqrt(var + np.float32(eps))).astype(np.float32)


def test_row_stats_three_partials_and_six_partial_mutant():
    rng = np.random.default_rng(2)
    y = (rng.standard_normal((64, H)) * 1.7 + 0.3).astype(np.float32)
    y += np.repeat(rng.standard_normal(H // 64) * 0.5, 64)[None, :].astype(np.float32)
    p = KR.partials(y).astype(np.float32)
    mean, rstd, mean_tol, rstd_rel = KR.stats_from_partials(p, 1e-12)
    m32, r32 = _row_stats32(p, 1e-12)
    KR.check("row_stats<3> mean", m32, mean, mean_tol)
    KR.check("row_stats<3> rstd", r32, rstd, rstd_rel * rstd)
    m6, r6 = _row_stats32(p, 1e-12, parts_read=6)
    with pytest.raises(AssertionError):
        KR.check("row_stats reading six partials", r6, rstd, rstd_rel * rstd)
