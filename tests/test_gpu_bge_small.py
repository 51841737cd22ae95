"""GPU: the bge-small geometry (BAAI/bge-small-en-v1.5: hidden 384, 12 heads of 32, inter 1536) on the CUDA path.

Kernel level, against the fp64 references of tests/kernel_refs.py and, for the head-dim-32 attention, tests/attention_refs.py,
at their named tolerances: the head-dim-32 attention, the
128-column GEMM tile for every epilogue (N = 384 / 1152; FFN1 at N = 1536 keeps the 256-column tile with 3 LayerNorm
partials), the residual epilogue's 3 partials, embed and pool_normalize on 384-wide rows; launch-shape invariance of the new
instantiations.  Model level, through the C ABI: parity with HF BertModel fp32 (tests/golden/bge_small_golden.npz) and the
numpy oracle layer by layer, batch invariance, bge-base and bge-small loaded side by side, and the router serving bge-small
from a hub snapshot."""
import importlib.util
import json
import os
import socket
import subprocess
import time
import urllib.request

import numpy as np
import pytest

import attention_refs as AR
import kernel_refs as KR
from oracle import bge_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "modal-examples_b200")
HD, H = 32, 384

REL_TOL = 1e-3
# "hard" weights (outlier channels, peaked attention, LayerNorm gains ~3): `tools/emulate_numerics.py --geometry small
# --style hard` (4 items x 512, 12 layers) puts the fp16-operand floor of this geometry at 5.7e-5 rel-L2 with fp32
# accumulation and exact softmax (6.1e-5 with fp16 P) -- below the hf style's 2.8e-4, and far below bge-base's 2.2e-3 that
# REL_TOL_HARD = 4e-3 in test_gpu_parity.py rests on.  So the hard cases keep the general 1e-3 bar here.
REL_TOL_HARD = 1e-3

_spec = importlib.util.spec_from_file_location("make_small_golden", os.path.join(ROOT, "tests", "golden", "make_small_golden.py"))
msg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(msg)


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


@pytest.fixture(scope="module")
def small_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "bge_small_golden.npz"))


_models = {}


def get_model(rt, layers, style, seed):
    key = (layers, style, seed)
    if key not in _models:
        g = msg.geometry(layers)
        flat = R.make_weights(g, seed, style)
        _models[key] = (g, flat, rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g)))
    return _models[key]


# ================================================================================================ attention, d = 32

def _qkv(rng, B, S, scale=2.0):
    return (rng.standard_normal((B * S, 3 * H)) * scale).astype(np.float16)


@pytest.mark.parametrize("S", [512, 511, 97])
def test_attention_d32_lens_on_every_sub_block_boundary(rt, S):
    lens = [n for n in [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 319, 320, 321, 383, 384, 385, 447, 448, 449, 511, 512]
            if n <= S] + [S]
    B = len(lens)
    qkv = _qkv(np.random.default_rng(S), B, S)
    ctx, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S, head_dim=HD)
    assert ctx.shape == (B * S, H)
    AR.check_attention(f"d=32 lens on sub-block boundaries, S={S}", ctx, qkv, lens, B, S, head_dim=HD)


def test_attention_d32_single_key_and_zero_queries(rt):
    B, S = 3, 200
    rng = np.random.default_rng(8)
    qkv = _qkv(rng, B, S, 3.0)
    ctx, _ = rt.debug_attention(qkv, np.ones(B, np.int32), B, S, head_dim=HD)
    v0 = qkv.reshape(B, S, 3 * H)[:, :1, 2 * H:]
    same = np.array_equal(ctx.reshape(B, S, H).view(np.uint16), np.broadcast_to(v0, (B, S, H)).view(np.uint16))
    print(f"d=32, len 1: every query row equals V[0] bitwise: {same}")
    assert same
    lens = [200, 129, 64]
    qkv[:, :H] = 0.0
    ctx, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S, head_dim=HD)
    v = qkv.reshape(B, S, 3 * H)[..., 2 * H:].astype(np.float64)
    mean = np.concatenate([np.broadcast_to(v[b, :n].mean(0), (S, H)) for b, n in enumerate(lens)])
    _, tol = AR.attention_ref(qkv, lens, B, S, head_dim=HD)
    KR.check("d=32, Q = 0: mean of the valid V rows", ctx, mean, tol)


def test_attention_d32_launch_shape_invariance(rt):
    """B = 4 (48 units): 1 / 2 / 7 / 47 / 48 CTAs walk (item, head) units, 49 / 66 / 131 / 132 walk query-tile units."""
    B, S, lens = 4, 512, [512, 77, 300, 129]
    qkv = _qkv(np.random.default_rng(4), B, S)
    base, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S, head_dim=HD)
    AR.check_attention("d=32 sms 0", base, qkv, lens, B, S, head_dim=HD)
    for sms in (1, 2, 7, 47, 48, 49, 66, 131, 132):
        got, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S, sms=sms, head_dim=HD)
        same = np.array_equal(got.view(np.uint16), base.view(np.uint16))
        print(f"d=32: sms {sms} ({'split by query tile' if B * 12 < sms else 'one unit per head'}) bitwise equal to sms 0: {same}")
        assert same, sms
    with pytest.raises(rt.B200RTError) as e:
        rt.debug_attention(qkv, np.array(lens, np.int32), B, S, head_dim=48)
    assert e.value.code == rt.E_INVALID


# ================================================================================================ GEMM, 128-column tile

def _ln_inputs(rng, M, W, mean=0.3, std=1.7):
    y = (rng.standard_normal((M, W)) * std + mean).astype(np.float32)
    y += np.repeat(rng.standard_normal(W // 64) * 0.5, 64)[None, :].astype(np.float32)
    g = (1.0 + 0.3 * rng.standard_normal(W)).astype(np.float32)
    b = (0.2 * rng.standard_normal(W)).astype(np.float32)
    return y, g, b


def _gemm_case(epi, M, N, K, seed, ln=True):
    """epi 0/1/3 fold a LayerNorm of the (K = 384 wide) A rows, epi 2 re-applies one to the (N = 384 wide) residual."""
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    kw = dict(eps=1e-12)
    if epi == 2:
        a = rng.standard_normal((M, K)).astype(np.float16)
        resid, g, b = _ln_inputs(rng, M, N, mean=-0.5, std=2.0)
        kw["resid"] = resid
        if ln:
            kw.update(ln_stats=KR.partials(KR.hilo64(*KR.split_hilo(resid))).astype(np.float32), ln_gamma=g, ln_beta=b)
    else:
        y, _, _ = _ln_inputs(rng, M, K)
        a = y.astype(np.float16)
        if ln:
            w = (w.astype(np.float32) - w.astype(np.float32).mean(1, keepdims=True)).astype(np.float16)
            kw["ln_stats"] = KR.partials(y).astype(np.float32)
    return (a, w, bias), kw


GEMM_CASES = [  # (epi, N, K): bge-small's QKV, FFN1 (256-column tile, 3 partials), attention-out and FFN2, and quick-GELU
    (0, 1152, 384), (1, 1536, 384), (2, 384, 384), (2, 384, 1536), (3, 384, 384)]


@pytest.mark.parametrize("M", [1, 127, 129, 300])
@pytest.mark.parametrize("epi,N,K", GEMM_CASES)
def test_gemm_small_geometry_epilogues(rt, epi, N, K, M):
    args, kw = _gemm_case(epi, M, N, K, seed=M * 7 + epi + N)
    if epi == 2:
        out, _, st = rt.debug_gemm(epi, *args, want_stats=True, **kw)
        KR.check_gemm(f"epi {epi} M={M} N={N} K={K}", out, epi, *args, **kw)
        assert st.shape == (M, 3, 2)
        KR.check_gemm_stats(f"epi {epi} M={M} N={N} K={K}: 3 partials", st, args, **kw)
    else:
        out, _ = rt.debug_gemm(epi, *args, **kw)
        KR.check_gemm(f"epi {epi} M={M} N={N} K={K}", out, epi, *args, **kw)


RESIDUAL_NO_LN_KS = [384, 1536]


@pytest.mark.parametrize("K", RESIDUAL_NO_LN_KS)
def test_residual_epilogue_three_partials_without_stats_in(rt, K):
    """stats_in = NULL (the residual added as is) at N = 384: 3 partials of the new rows, including rows of mean 150."""
    M, N = 300, 384
    rng = np.random.default_rng(K)
    a = rng.standard_normal((M, K)).astype(np.float16)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = (0.1 * rng.standard_normal(N)).astype(np.float32)
    resid = (rng.standard_normal((M, N)) * 2.0).astype(np.float32)
    resid[::3] = (150.0 + rng.standard_normal((len(resid[::3]), N))).astype(np.float32)
    out, _, st = rt.debug_gemm(2, a, w, bias, resid, want_stats=True)
    KR.check_gemm(f"N=384 K={K} residual, no LayerNorm", out, 2, a, w, bias, resid=resid)
    KR.check_gemm_stats(f"N=384 K={K} residual, no LayerNorm: stats_out", st, (a, w, bias), resid=resid)


@pytest.mark.parametrize("epi,N,K", [(0, 1152, 384), (2, 384, 1536)])
def test_gemm_small_geometry_launch_shape_invariance(rt, epi, N, K):
    """297 tiles (33 x 9, QKV) / 97 tiles (FFN2), the last row tile partly filled, on 1, 2, 7, 66, 131, 132 CTAs: outputs
    and statistics bitwise equal to the launch on every SM.  K = 1536 is 24 k-blocks through the 4-stage ring."""
    M = 4100 if epi == 0 else 12300
    args, kw = _gemm_case(epi, M, N, K, seed=30 + epi)
    want = epi == 2
    base = rt.debug_gemm(epi, *args, want_stats=want, **kw)
    KR.check_gemm(f"epi {epi} N={N} sms 0", base[0], epi, *args, **kw)
    for sms in (1, 2, 7, 66, 131, 132):
        got = rt.debug_gemm(epi, *args, want_stats=want, sms=sms, **kw)
        view = np.uint32 if epi == 2 else np.uint16
        same = np.array_equal(got[0].view(view), base[0].view(view))
        same_st = not want or np.array_equal(got[2].view(np.uint32), base[2].view(np.uint32))
        print(f"epi {epi} N={N}: sms {sms} bitwise equal to sms 0: out {same}, stats {same_st}")
        assert same and same_st, sms


def test_gemm_rejects_other_layernorm_widths(rt):
    args, kw = _gemm_case(0, 64, 512, 512, seed=1, ln=False)
    kw["ln_stats"] = np.zeros((64, 4, 2), np.float32)
    with pytest.raises(rt.B200RTError) as e:
        rt.debug_gemm(0, *args, **kw)
    assert e.value.code == rt.E_INVALID


# ================================================================================================ row kernels at 384

def test_embed_width_384(rt):
    vocab, S, n_items = 64, 100, 3
    rng = np.random.default_rng(5)
    word = (rng.standard_normal((vocab, H)) + np.repeat(rng.standard_normal(3) * 3.0, 128)[None, :]).astype(np.float32)
    pos = rng.standard_normal((S, H)).astype(np.float32)
    type0 = (0.3 * rng.standard_normal(H)).astype(np.float32)
    word[1, :16] = -0.0
    pos[:, :16] = -0.0
    type0[:16] = -0.0
    word[3, :8] = [70000, -70000, 65520, 65519, 2.0 ** -25, 3e-8, 1 + 2.0 ** -11, 0.0]
    ids = rng.integers(0, vocab, size=n_items * S).astype(np.int32)
    ids[:4] = [1, 3, 0, vocab - 1]
    hi, lo, st = rt.debug_embed(ids, word, pos, type0, S, hidden=H)
    assert hi.shape == (n_items * S, H) and st.shape == (n_items * S, 3, 2)
    KR.check_embed("embed 384", hi, lo, st, ids, word, pos, type0, S)


@pytest.mark.parametrize("S,n_items", [(1, 5), (7, 133), (512, 9)])
def test_pool_normalize_width_384(rt, S, n_items):
    rng = np.random.default_rng(S + 1)
    hi, lo = KR.split_hilo((rng.standard_normal((n_items * S, H)) * 1.5 + 0.4).astype(np.float32))
    g = (1.0 + 0.3 * rng.standard_normal(H)).astype(np.float32)
    b = (0.2 * rng.standard_normal(H)).astype(np.float32)
    out = rt.debug_pool_normalize(hi, lo, g, b, S, 1e-12, hidden=H)
    KR.check_pool_normalize(f"pool_normalize 384 S={S} n={n_items}", out, hi, lo, g, b, S, 1e-12)
    hi[0], lo[0] = np.float16(3.25), np.float16(2.0 ** -12)  # a constant CLS row, beta = 0: zeros, as F.normalize gives
    out = rt.debug_pool_normalize(hi, lo, g, np.zeros(H, np.float32), S, 1e-12, hidden=H)
    assert np.isfinite(out).all() and (out[0] == 0.0).all(), out[0][:8]


def test_fold_ln_at_small_widths(rt):
    rng = np.random.default_rng(7)
    for N, K in ((1152, 384), (384, 1536)):
        w = (rng.standard_normal((N, K)) * 0.04).astype(np.float32)
        g = (1.0 + 0.3 * rng.standard_normal(K)).astype(np.float32)
        b = (0.2 * rng.standard_normal(K)).astype(np.float32)
        bias = rng.standard_normal(N).astype(np.float32)
        w_out, cvec = rt.debug_fold_ln(w, g, b, bias)
        KR.check_fold_ln(f"fold_ln N={N} K={K}", w_out, cvec, w, g, b, bias)


# ================================================================================================ model level

@pytest.mark.parametrize("case", list(msg.CASES))
def test_embeddings_vs_small_golden(rt, small_golden, case):
    layers, style, wseed, spec = msg.CASES[case]
    g, flat, model = get_model(rt, layers, style, wseed)
    ids, lens = msg.case_inputs(spec)
    emb = model.embed(ids, lens)
    assert emb.shape == (ids.shape[0], H)
    rel = R.rel_l2(emb, small_golden[f"{case}_emb"])
    print(f"bge-small case {case} ({style}, {layers} layers): max rel-L2 vs HF fp32 {rel.max():.3e}")
    assert rel.max() <= (REL_TOL_HARD if style == "hard" else REL_TOL), rel
    assert np.allclose(np.linalg.norm(emb, axis=1), 1.0, atol=1e-5)


def test_residual_stream_layer_by_layer(rt):
    g, flat, model = get_model(rt, 12, "trained", 0)
    ids, lens = R.synth_ragged(3, 160, seed=9, min_len=20)
    _, hidden = R.forward_np(flat, ids, lens, g, return_hidden=True)
    for L in (0, 1, 2, 6, 12):
        # the oracle's hidden state: the LayerNorm that holds after layer L, applied in fp64 to the residual stream
        ln = ("emb.ln.g", "emb.ln.b") if L == 0 else (f"l{L - 1}.ln2.g", f"l{L - 1}.ln2.b")
        h = KR.layernorm_ref(model.debug_residual(ids, lens, L), flat[ln[0]], flat[ln[1]], g.eps)[0]
        assert h.shape == (3, 160, H)
        for i, n in enumerate(lens):
            d = h[i, :n] - hidden[L][i, :n]
            rel = np.sqrt((d ** 2).sum()) / np.sqrt((hidden[L][i, :n] ** 2).sum())
            assert rel < (1e-6 if L == 0 else REL_TOL), (L, i, rel)


def test_batch_invariance(rt):
    """An item's embedding is bitwise the same alone, in a ragged batch and in a full 132-item wave of 512 tokens."""
    g, flat, model = get_model(rt, 12, "hf", 0)
    n = rt.wave_capacity_items()
    ids, lens = R.synth_ragged(n, 512, seed=21, min_len=449)  # one 512-token bucket: one full wave
    full = model.embed(ids, lens)
    ref = R.forward_np(flat, ids[:2], lens[:2], g)
    assert R.rel_l2(full[:2], ref).max() <= REL_TOL
    for k in (0, 5, n - 1):
        alone = model.embed(ids[k:k + 1, :lens[k]], lens[k:k + 1])
        rag_ids, rag_lens = R.synth_ragged(9, 512, seed=22 + k, min_len=1)
        rag_ids[4, :] = ids[k]
        rag_lens[4] = lens[k]
        ragged = model.embed(rag_ids, rag_lens)
        same = np.array_equal(alone[0].view(np.uint32), full[k].view(np.uint32)) and np.array_equal(ragged[4].view(np.uint32), full[k].view(np.uint32))
        print(f"item {k} (len {lens[k]}): alone / ragged batch / full wave bitwise equal: {same}")
        assert same, k


def test_two_geometries_in_one_runtime(rt):
    """bge-base and bge-small loaded side by side, submissions interleaved: each output is bitwise the output of that model
    loaded alone in a runtime of its own.  The module's runtime is restarted for the duration."""
    bg = R.BertGeometry(layers=2)
    sg = msg.geometry(2)
    bblob = R.pack_blob(R.make_weights(bg, 3, "trained"), bg)
    sblob = R.pack_blob(R.make_weights(sg, 3, "trained"), sg)
    inputs = [R.synth_ragged(int(n), int(S), seed=300 + i, min_len=1) for i, (n, S) in enumerate([(5, 64), (17, 512), (3, 200), (40, 128)])]

    def alone(geom, blob):
        rt.shutdown()
        rt.init(devices=[0])
        m = rt.EmbedModel(R.geometry_dict(geom), blob)
        return [m.embed(i, l) for i, l in inputs]

    try:
        want_b = alone(bg, bblob)
        want_s = alone(sg, sblob)
        rt.shutdown()
        rt.init(devices=[0])
        mb = rt.EmbedModel(R.geometry_dict(bg), bblob)
        ms = rt.EmbedModel(R.geometry_dict(sg), sblob)
        tickets = []
        for k, (i, l) in enumerate(inputs):
            tickets.append((ms, "small", k, ms.submit(i, l)))
            tickets.append((mb, "base", k, mb.submit(i, l)))
        for m, name, k, t in tickets:
            got = m.wait(t, 120_000)
            want = (want_s if name == "small" else want_b)[k]
            assert got.shape == want.shape == (inputs[k][0].shape[0], 384 if name == "small" else 768)
            same = np.array_equal(got.view(np.uint32), want.view(np.uint32))
            print(f"{name} input {k}: interleaved == loaded alone bitwise: {same}")
            assert same, (name, k)
    finally:
        _models.clear()
        rt.shutdown()
        rt.init(devices=[0])


def test_other_geometries_stay_unsupported(rt):
    g = msg.geometry(1)
    flat = R.make_weights(g, 0, "hf")
    for bad in (dict(hidden=1024), dict(heads=6), dict(inter=3072)):
        with pytest.raises(rt.B200RTError) as e:
            rt.EmbedModel(dict(R.geometry_dict(g), **bad), R.pack_blob(flat, g))
        assert e.value.code == rt.E_UNSUPPORTED
        assert "bge-base" in str(e.value) and "bge-small" in str(e.value), str(e.value)


# ================================================================================================ router

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_router_serves_bge_small_from_a_hub_snapshot(tmp_path):
    """A hub snapshot of seeded bge-small weights (model.safetensors + config.json); the router started the way the reference
    starts TEI returns 384-vectors within 1e-3 of HF BertModel fp32 on the router's own tokenization."""
    import torch
    from b200rt import weights as W
    from tei_router.tokenizer import WordPiece

    g = msg.geometry(12)
    flat = R.make_weights(g, 5, "trained")
    snap = tmp_path / "models--BAAI--bge-small-en-v1.5" / "snapshots" / "0123abc"
    snap.mkdir(parents=True)
    W.write_safetensors(str(snap / "model.safetensors"), {k: np.ascontiguousarray(v, np.float32) for k, v in R.flat_to_hf_state(flat, g).items()})
    (snap / "config.json").write_text(json.dumps({"hidden_size": 384, "num_attention_heads": 12, "intermediate_size": 1536,
                                                  "layer_norm_eps": 1e-12}))
    port = _free_port()
    env = dict(os.environ, PATH=os.path.join(PKG, "bin") + os.pathsep + os.environ["PATH"], B200RT_GPUS="1")
    proc = subprocess.Popen(["text-embeddings-router", "--model-id", "BAAI/bge-small-en-v1.5", "--port", str(port),
                             "--huggingface-hub-cache", str(tmp_path)], env=env)
    try:
        deadline = time.time() + 300
        while True:
            try:
                socket.create_connection(("127.0.0.1", port), timeout=1).close()
                break
            except OSError:
                assert proc.poll() is None, f"launcher exited unexpectedly with code {proc.returncode}"
                assert time.time() < deadline, "router did not become ready"
                time.sleep(0.2)
        texts = [f"Wikipedia paragraph {i}: {'the quick brown fox ' * (i % 9)}jumps over the lazy dog." for i in range(24)]
        req = urllib.request.Request(f"http://127.0.0.1:{port}/embed", data=json.dumps({"inputs": texts}).encode(),
                                     headers={"Content-Type": "application/json"})
        with urllib.request.urlopen(req, timeout=120) as r:
            assert r.status == 200
            out = json.loads(r.read())
    finally:
        proc.terminate()
        proc.wait(timeout=60)
    got = np.array(out, np.float32)
    assert got.shape == (24, 384)
    tok = WordPiece()
    rows = [tok.encode(t, 512, True) for t in texts]
    lens = np.array([len(r) for r in rows], np.int32)
    ids = np.zeros((len(rows), int(lens.max())), np.int32)
    for i, r in enumerate(rows):
        ids[i, : len(r)] = r
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    ref = R.forward_hf(R.build_hf_model(flat, g), ids, lens)
    rel = R.rel_l2(got, ref)
    print(f"router bge-small: max rel-L2 vs HF fp32 {rel.max():.3e}")
    assert rel.max() <= REL_TOL
