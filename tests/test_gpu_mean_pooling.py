"""GPU (`-m gpu`): mean pooling (B200RT_LOAD_POOL_MEAN; sentence-transformers Pooling(mean) + Normalize, the pooling of
all-MiniLM-L6-v2, e5 and gte).  Kernel conformance of mean_pool_normalize against its fp64 reference, the forward chain of a
mean model against the CLS model of the same weights, parity with HF fp32 (tests/golden/minilm_golden.npz) and the fp64
oracle, bitwise invariance of an item's embedding across batches, launch paths and replicas, CLS and mean models side by
side, and the router serving a MiniLM hub snapshot."""
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
import mean_pool_refs as MP
from oracle import bge_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "modal-examples_b200")

REL_TOL = 1e-3
# "hard" weights (outlier channels, peaked attention, LayerNorm gains ~3), 12-layer bge-base geometry, mean pooling:
# `tools/emulate_numerics.py --style hard --pooling mean` (these 4 items x 512, lengths >= 128, fp16 operands, fp32
# accumulation) puts the fp16-operand floor of the shipped design (LayerNorm folded into the GEMMs, fp16 P) at 7.6e-4 rel-L2
# against fp64 (7.4e-4 with exact P).  Averaging over the tokens keeps it below the CLS row's 2.2e-3 on the same weights,
# which test_gpu_parity.py's 4e-3 rests on; the bar leaves the same ~2.5x for the kernels' own fp32 rounding.
REL_TOL_HARD_MEAN = 2e-3

_spec = importlib.util.spec_from_file_location("make_minilm_golden", os.path.join(ROOT, "tests", "golden", "make_minilm_golden.py"))
mmg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mmg)


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ================================================================================================ kernel conformance

LENS = [1, 2, 7, 63, 64, 65, 127, 128, 511, 512]


def _rows(rng, n_rows, W):
    x = rng.standard_normal((n_rows, W)).astype(np.float32) * 2.0 + 0.3
    x[:, :3] *= 20.0
    return KR.split_hilo(x)


def _ln(rng, W):
    return (1.0 + 0.2 * rng.standard_normal(W)).astype(np.float32), (0.1 * rng.standard_normal(W)).astype(np.float32)


def _fill_padding(hi, lo, lens, S, how, rng):
    hi, lo = hi.copy(), lo.copy()
    W = hi.shape[1]
    for i, n in enumerate(lens):
        n = int(min(max(n, 1), S))
        if n == S:
            continue
        sl = slice(i * S + n, (i + 1) * S)
        if how == "zeros":
            hi[sl] = 0
            lo[sl] = 0
        else:  # NaN and +-65504 (fp16 max)
            vals = np.array([np.nan, 65504.0, -65504.0], np.float16)
            hi[sl] = vals[rng.integers(0, 3, size=(S - n, W))]
            lo[sl] = vals[rng.integers(0, 3, size=(S - n, W))]
    return hi, lo


@pytest.mark.parametrize("W", [384, 768])
@pytest.mark.parametrize("S,B", [(64, 132), (128, 40), (512, 12)])
def test_mean_pool_kernel_conformance(rt, W, S, B):
    """Within the fp64 reference's tolerance for every length on and around the 8-row and 64-row steps; rows past len hold
    NaN / +-65504 and the result is finite and bitwise the result with zeros there."""
    rng = np.random.default_rng(W * 1000 + S)
    base = [n for n in LENS if n <= S] + [S]
    lens = np.array([base[i % len(base)] if i < len(base) else int(rng.integers(1, S + 1)) for i in range(B)], np.int32)
    hi, lo = _rows(rng, B * S, W)
    g, b = _ln(rng, W)
    hz, lz = _fill_padding(hi, lo, lens, S, "zeros", rng)
    hp, lp = _fill_padding(hi, lo, lens, S, "poison", rng)
    out_z = rt.debug_mean_pool_normalize(hz, lz, g, b, lens, S, 1e-12, hidden=W)
    out_p = rt.debug_mean_pool_normalize(hp, lp, g, b, lens, S, 1e-12, hidden=W)
    assert np.isfinite(out_p).all()
    assert np.array_equal(_bits(out_z), _bits(out_p)), "padding rows changed the result"
    MP.check_mean_pool_normalize(f"mean_pool W={W} S={S} B={B}", out_z, hz, lz, g, b, lens, S, 1e-12)
    assert np.allclose(np.linalg.norm(out_z, axis=1), 1.0, atol=1e-5)


@pytest.mark.parametrize("W", [384, 768])
def test_mean_pool_kernel_clamps_device_lengths(rt, W):
    """Lengths 0, negative and > S (device lengths nothing validates) are clamped to [1, S]: the result is the clamped
    length's, and the neighbouring items' rows -- poisoned -- are never read."""
    rng = np.random.default_rng(W + 7)
    S = 64
    lens_bad = np.array([0, -5, S + 1, 1 << 30, 5], np.int32)
    lens_ok = np.clip(lens_bad, 1, S).astype(np.int32)
    B = len(lens_bad)
    hi, lo = _rows(rng, B * S, W)
    hi, lo = _fill_padding(hi, lo, lens_ok, S, "poison", rng)  # a read past any item's clamped length meets NaN
    g, b = _ln(rng, W)
    got = rt.debug_mean_pool_normalize(hi, lo, g, b, lens_bad, S, 1e-12, hidden=W)
    want = rt.debug_mean_pool_normalize(hi, lo, g, b, lens_ok, S, 1e-12, hidden=W)
    assert np.isfinite(got).all()
    assert np.array_equal(_bits(got), _bits(want))
    MP.check_mean_pool_normalize(f"clamped W={W}", got, hi, lo, g, b, lens_bad, S, 1e-12)


def test_mean_pool_kernel_is_batch_invariant(rt):
    """An item's result does not depend on B, S (its padding) or its position in the batch."""
    rng = np.random.default_rng(5)
    W, n = 384, 77
    x_hi, x_lo = _rows(rng, n, W)
    g, b = _ln(rng, W)
    outs = []
    for S, B, pos in ((77, 1, 0), (128, 9, 4), (512, 3, 2)):
        hi, lo = _rows(rng, B * S, W)
        hi[pos * S:pos * S + n], lo[pos * S:pos * S + n] = x_hi, x_lo
        lens = rng.integers(1, S + 1, size=B).astype(np.int32)
        lens[pos] = n
        outs.append(rt.debug_mean_pool_normalize(hi, lo, g, b, lens, S, 1e-12, hidden=W)[pos])
    assert all(np.array_equal(_bits(o), _bits(outs[0])) for o in outs[1:])


# ================================================================================================ models

_models = {}


def get_model(rt, g, style, seed, pooling):
    key = (g, style, seed, pooling)
    if key not in _models:
        flat = R.make_weights(g, seed, style)
        _models[key] = (flat, rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g), pooling=pooling))
    return _models[key]


def test_load_flags(rt):
    import ctypes

    g = mmg.geometry()
    flat = R.make_weights(R.BertGeometry(layers=1, hidden=384, heads=12, inter=1536), 0, "hf")
    blob = R.pack_blob(flat, R.BertGeometry(layers=1, hidden=384, heads=12, inter=1536))
    cfg = rt.BertConfig(g.vocab, 384, 1, 12, 1536, 512, 2, 1e-12)
    lib = rt.load_library()
    h = ctypes.c_int32(-1)
    assert lib.b200rt_model_load_ex(b"bert", ctypes.byref(cfg), rt._ptr(blob), blob.nbytes, 2, ctypes.byref(h)) == rt.E_INVALID
    vcfg = rt.VitConfig(224, 16, 768, 1, 12, 3072, 512, 1e-5)
    assert lib.b200rt_model_load_ex(b"vit", ctypes.byref(vcfg), rt._ptr(blob), blob.nbytes, 1, ctypes.byref(h)) == rt.E_INVALID
    assert b"vit" in lib.b200rt_last_error()
    assert lib.b200rt_model_load_ex(b"bert", ctypes.byref(cfg), rt._ptr(blob), blob.nbytes, 1, ctypes.byref(h)) == 0


def test_forward_chain_differs_from_cls_only_in_the_pool(rt):
    """2-layer mean and CLS models of the same weights: launches 1 .. 5L + 1 leave bitwise the same workspace; the last
    launch is mean_pool_normalize and passes the kernel check on the traced hi / lo, with the last layer's LN2."""
    for g in (R.BertGeometry(layers=2), R.BertGeometry(layers=2, hidden=384, heads=12, inter=1536)):
        flat, mean = get_model(rt, g, "trained", 3, "mean")
        _, cls = get_model(rt, g, "trained", 3, "cls")
        ids, lens = R.synth_ragged(5, 96, seed=31, min_len=1)
        lens[0] = 1
        tm = mean.debug_trace(ids, lens, 5 * g.layers + 2)
        tc = cls.debug_trace(ids, lens, 5 * g.layers + 2)
        assert tm["n_total"] == tc["n_total"] == 5 * g.layers + 2
        assert tm["names"][:-1] == tc["names"][:-1]
        assert tm["names"][-1] == "mean_pool_normalize" and tc["names"][-1] == "pool_normalize"
        for k in ("yhi", "ylo", "pstats0", "pstats1", "qkv", "ctx", "ffn"):
            assert np.array_equal(tm[k].view(np.uint8), tc[k].view(np.uint8)), k
        M, S = tm["M"], ids.shape[1]
        last = f"l{g.layers - 1}.ln2."
        MP.check_mean_pool_normalize(f"traced mean pool H={g.hidden}", tm["out"], tm["yhi"][:M], tm["ylo"][:M],
                                     flat[last + "g"], flat[last + "b"], lens, S, g.eps)
        assert np.array_equal(_bits(mean.embed(ids, lens)), _bits(tm["out"]))
        profile = mean.profile_forward(4, 128, iters=1)
        assert "mean_pool_normalize" in profile and "pool_normalize" not in profile


# ================================================================================================ parity

@pytest.mark.parametrize("case", list(mmg.CASES))
def test_minilm_vs_golden(rt, case):
    style, seed, spec = mmg.CASES[case]
    g = mmg.geometry()
    _, model = get_model(rt, g, style, seed, "mean")
    ids, lens = mmg.case_inputs(spec)
    emb = model.embed(ids, lens)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "minilm_golden.npz"))[f"{case}_emb"]
    rel = R.rel_l2(emb, gold)
    print(f"MiniLM-L6 case {case} ({style}): max rel-L2 vs HF fp32 mean pooling {rel.max():.3e}")
    assert emb.shape == (ids.shape[0], 384) and rel.max() <= REL_TOL, rel


@pytest.mark.parametrize("style,bar", [("trained", REL_TOL), ("hard", REL_TOL_HARD_MEAN)])
def test_bge_base_geometry_mean_vs_fp64_oracle(rt, style, bar):
    """12-layer bge-base geometry (the shape of gte-base / e5-base) with mean pooling against the fp64 oracle."""
    g = R.BertGeometry()
    flat, model = get_model(rt, g, style, 0, "mean")
    ids, lens = R.synth_ragged(4, 512, seed=1, min_len=128)  # the inputs emulate_numerics runs
    emb = model.embed(ids, lens)
    ref = MP.forward_np_mean(flat, ids, lens, g)
    rel = R.rel_l2(emb, ref)
    print(f"bge-base geometry, mean pooling, {style}: max rel-L2 vs fp64 {rel.max():.3e} (bar {bar:g})")
    assert rel.max() <= bar, rel


# ================================================================================================ invariance

def test_item_is_bitwise_invariant_across_batches_and_launch_paths(rt):
    """alone / in a ragged batch of another bucket / in a graph-replayed batch (<= 8192 rows) / in a plain-launch batch /
    through embed_device: the same bits."""
    import torch

    g = mmg.geometry()
    _, model = get_model(rt, g, "trained", 3, "mean")
    ids, lens = R.synth_ragged(40, 256, seed=41, min_len=1)
    lens[:4] = [1, 2, 65, 256]
    # plain launches: 40 x 256 = 10240 rows > 8192; graph replay: 8 x 256 = 2048 rows
    big = model.embed(ids, lens)
    small = model.embed(ids[:8], lens[:8])
    assert np.array_equal(_bits(big[:8]), _bits(small))
    for k in range(4):
        alone = model.embed(ids[k:k + 1, :lens[k]], lens[k:k + 1])
        rag_ids, rag_lens = R.synth_ragged(7, 512, seed=50 + k, min_len=300)  # a 512-token bucket
        rag_ids[3] = 0
        rag_ids[3, :lens[k]] = ids[k, :lens[k]]
        rag_lens[3] = lens[k]
        ragged = model.embed(rag_ids, rag_lens)
        assert np.array_equal(_bits(alone[0]), _bits(big[k])), k
        assert np.array_equal(_bits(ragged[3]), _bits(big[k])), k
    with torch.cuda.device(0):
        d_ids, d_lens = torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda()
        d_out = torch.empty((40, 384), dtype=torch.float32, device="cuda")
        st = torch.cuda.Stream()
        model.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), 40, 256, d_out.data_ptr(), st.cuda_stream)  # plain
        model.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), 8, 256, d_out.data_ptr(), st.cuda_stream)   # graph
        st.synchronize()
        dev = d_out.cpu().numpy()
    assert np.array_equal(_bits(dev), _bits(big))


def test_cls_and_mean_side_by_side(rt):
    """CLS and mean models of the same weights loaded together: the CLS model's outputs are bitwise those of the same model
    loaded alone, each model's graphs are its own, and a forward costs 5L + 2 launches for both (+1 scatter per wave)."""
    import torch

    g = mmg.geometry()
    flat = R.make_weights(g, 3, "trained")
    blob = R.pack_blob(flat, g)
    inputs = [R.synth_ragged(n, S, seed=60 + n, min_len=1) for n, S in ((5, 64), (3, 200), (17, 512))]
    try:
        rt.shutdown()
        rt.init(devices=[0])
        alone = [rt.EmbedModel(R.geometry_dict(g), blob).embed(i, l) for i, l in inputs]
        rt.shutdown()
        rt.init(devices=[0])
        cls = rt.EmbedModel(R.geometry_dict(g), blob, pooling="cls")
        mean = rt.EmbedModel(R.geometry_dict(g), blob, pooling="mean")
        tickets = []
        for k, (i, l) in enumerate(inputs):
            tickets.append(("mean", k, mean.submit(i, l)))
            tickets.append(("cls", k, cls.submit(i, l)))
        got = {}
        for name, k, t in tickets:
            got[(name, k)] = (mean if name == "mean" else cls).wait(t, 120_000)
        for k in range(len(inputs)):
            assert np.array_equal(_bits(got[("cls", k)]), _bits(alone[k])), k
            assert not np.array_equal(_bits(got[("mean", k)]), _bits(alone[k])), k
            ref = MP.forward_np_mean(flat, *inputs[k], g)
            assert R.rel_l2(got[("mean", k)], ref).max() <= REL_TOL
        ids, lens = inputs[0]
        with torch.cuda.device(0):
            d_ids, d_lens = torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda()
            d_out = torch.empty((len(ids), 384), dtype=torch.float32, device="cuda")
            for m in (cls, mean, cls, mean):  # the same (buffers, shape) for both models: each replays its own graph
                n0 = rt.stats()["kernel_launches"]
                m.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), len(ids), ids.shape[1], d_out.data_ptr(), 0)
                rt.device_sync(0)
                assert rt.stats()["kernel_launches"] - n0 == 5 * g.layers + 2
                want = got[("cls" if m is cls else "mean", 0)]
                assert np.array_equal(_bits(d_out.cpu().numpy()), _bits(want))
        for m in (cls, mean):
            n0 = rt.stats()["kernel_launches"]
            m.embed(ids[:1], lens[:1])  # one item, one wave: the forward + the wave's scatter
            assert rt.stats()["kernel_launches"] - n0 == 5 * g.layers + 2 + 1
    finally:
        _models.clear()
        rt.shutdown()
        rt.init(devices=[0])


def test_replicas_and_split_sm_runtime_give_the_same_bits(rt):
    """Every replica of a min(visible, 8) pool, and the split-SM runtime (k = 21, two replicas on one GPU), give the bits of
    the one-replica runtime."""
    import torch

    g = mmg.geometry()
    blob = R.pack_blob(R.make_weights(g, 3, "trained"), g)
    ids, lens = R.synth_ragged(40, 192, seed=71, min_len=129)  # one bucket: spread over every replica
    ids2 = R.synth_ids(2, 64, 5)

    def run(n=None, devices=None, flags=0):
        rt.shutdown()
        if devices is not None:
            rt.init(devices=devices, flags=flags)
        else:
            rt.init(n)
        m = rt.EmbedModel(R.geometry_dict(g), blob, pooling="mean")
        G = rt.num_gpus()
        small = [m.embed(ids2) for _ in range(2 * G + 1)]  # consecutive small waves rotate over the replicas
        return m.embed(ids, lens), small, G, rt.stats()["peer_bytes"]

    try:
        one, small1, _, _ = run(devices=[0])
        pool, small_p, G, _ = run(n=min(torch.cuda.device_count(), 8))
        split, small_s, G2, peer = run(devices=[0], flags=rt.SPLIT_SMS(21))
    finally:
        _models.clear()
        rt.shutdown()
        rt.init(devices=[0])
    assert G2 == 2 and peer > 0
    print(f"replicas in the pool: {G}")
    for name, a, sm in (("pool", pool, small_p), ("split k=21", split, small_s)):
        assert np.array_equal(_bits(a), _bits(one)), name
        assert all(np.array_equal(_bits(s), _bits(small1[0])) for s in sm), name


# ================================================================================================ router

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _minilm_snapshot(tmp_path, flat, g):
    from b200rt import weights as W

    snap = tmp_path / "models--sentence-transformers--all-MiniLM-L6-v2" / "snapshots" / "7dbbc90"
    (snap / "1_Pooling").mkdir(parents=True)
    W.write_safetensors(str(snap / "model.safetensors"), {k: np.ascontiguousarray(v, np.float32) for k, v in R.flat_to_hf_state(flat, g).items()})
    (snap / "config.json").write_text(json.dumps({"hidden_size": 384, "num_attention_heads": 12, "intermediate_size": 1536,
                                                  "num_hidden_layers": 6, "layer_norm_eps": 1e-12}))
    (snap / "modules.json").write_text(json.dumps([
        {"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
        {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
        {"idx": 2, "name": "2", "path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}]))
    (snap / "1_Pooling" / "config.json").write_text(json.dumps({
        "word_embedding_dimension": 384, "pooling_mode_cls_token": False, "pooling_mode_mean_tokens": True,
        "pooling_mode_max_tokens": False, "pooling_mode_mean_sqrt_len_tokens": False}))


def _start_router(tmp_path, extra):
    port = _free_port()
    env = dict(os.environ, PATH=os.path.join(PKG, "bin") + os.pathsep + os.environ["PATH"], B200RT_GPUS="1")
    proc = subprocess.Popen(["text-embeddings-router", "--model-id", "sentence-transformers/all-MiniLM-L6-v2", "--port", str(port),
                             "--huggingface-hub-cache", str(tmp_path)] + extra, env=env)
    deadline = time.time() + 300
    while True:
        try:
            socket.create_connection(("127.0.0.1", port), timeout=1).close()
            return proc, port
        except OSError:
            if proc.poll() is not None:
                return proc, None
            assert time.time() < deadline, "router did not become ready"
            time.sleep(0.2)


def _embed_and_info(port, texts):
    req = urllib.request.Request(f"http://127.0.0.1:{port}/embed", data=json.dumps({"inputs": texts}).encode(),
                                 headers={"Content-Type": "application/json"})
    with urllib.request.urlopen(req, timeout=120) as r:
        out = np.array(json.loads(r.read()), np.float32)
    with urllib.request.urlopen(f"http://127.0.0.1:{port}/info", timeout=10) as r:
        info = json.loads(r.read())
    return out, info


def test_router_serves_minilm_mean_pooled_from_a_hub_snapshot(tmp_path):
    import torch
    from tei_router.tokenizer import WordPiece

    g = mmg.geometry()
    flat = R.make_weights(g, 5, "trained")
    _minilm_snapshot(tmp_path, flat, g)
    texts = [f"Sentence {i}: {'a sentence transformer ' * (i % 6)}pools the mean of its tokens." for i in range(20)]
    tok = WordPiece()
    rows = [tok.encode(t, 512, True) for t in texts]
    lens = np.array([len(r) for r in rows], np.int32)
    ids = np.zeros((len(rows), int(lens.max())), np.int32)
    for i, r in enumerate(rows):
        ids[i, : len(r)] = r
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    hf = R.build_hf_model(flat, g)
    results = {}
    for extra, name in (([], "declared"), (["--pooling", "cls"], "cls")):
        proc, port = _start_router(tmp_path, extra)
        try:
            assert port is not None, f"router exited with code {proc.returncode}"
            results[name] = _embed_and_info(port, texts)
        finally:
            proc.terminate()
            proc.wait(timeout=60)
    got, info = results["declared"]
    assert got.shape == (20, 384) and info["pooling"] == "mean"
    rel = R.rel_l2(got, MP.forward_hf_mean(hf, ids, lens))
    print(f"router MiniLM-L6 (mean): max rel-L2 vs HF fp32 mean pooling {rel.max():.3e}")
    assert rel.max() <= REL_TOL
    got_cls, info_cls = results["cls"]
    assert info_cls["pooling"] == "cls"
    assert R.rel_l2(got_cls, R.forward_hf(hf, ids, lens)).max() <= REL_TOL
    # an unsupported --pooling: non-zero exit before the port is bound
    proc, port = _start_router(tmp_path, ["--pooling", "splade"])
    proc.wait(timeout=120)
    assert port is None and proc.returncode != 0
