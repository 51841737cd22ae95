"""CPU: nomic-bert (kind "nomic_bert") -- the fp64 oracle against HF NomicBertModel, the weight loaders and config reader,
the kernel references against their emulations and the wiring mutants they must reject, and the emulated fp16-operand floor
that the GPU parity bars (nomic_refs.BARS) stand on, recorded by the HF golden's generator and asserted here."""
import json
import os

import numpy as np
import pytest

import kernel_refs as KR
import nomic_refs as N
from b200rt import weights as W

G2 = N.geometry(layers=2, max_pos=2048)


def _rel(a, b):
    return np.linalg.norm(np.asarray(a, np.float64) - b, axis=-1) / np.linalg.norm(b, axis=-1)


def _ids(rng, lens, S):
    ids = np.zeros((len(lens), S), np.int32)
    for i, n in enumerate(lens):
        ids[i, :n] = rng.integers(1000, 30528, n)
    return ids


# ------------------------------------------------------------------------------------------------ oracle

@pytest.mark.parametrize("style", ["hf", "trained"])
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_oracle_matches_hf(style, pooling):
    pytest.importorskip("transformers")
    flat = N.make_weights(G2, 3, style)
    lens = [600, 77, 5]
    ids = _ids(np.random.default_rng(0), lens, 600)
    ref = N.forward_np(flat, ids, lens, G2, pooling)
    hf = N.forward_hf(N.build_hf_model(flat, G2), ids, lens, pooling)
    rel = _rel(hf, ref)
    print(f"oracle vs HF fp32 ({style}, {pooling}): {rel.max():.2e}")
    assert rel.max() <= 5e-6


def test_hf_style_is_random_nomic_blob():
    assert (N.pack(N.make_weights(G2, 4, "hf"), G2).view(np.uint32) == W.random_nomic_blob(G2, 4).view(np.uint32)).all()


def test_rotary_positions_matter():
    """Rotary scores depend on position differences only: shifting every position leaves the embeddings as they are (to
    rounding), while dropping the rotation moves them by far more than the GPU parity bar."""
    flat = N.make_weights(G2, 3, "trained")
    lens = [300, 40]
    ids = _ids(np.random.default_rng(1), lens, 300)
    ref = N.forward_np(flat, ids, lens, G2)
    assert _rel(N.forward_np(flat, ids, lens, G2, shift=1), ref).max() < 1e-6
    moved = _rel(N.forward_np(flat, ids, lens, G2, rope=False), ref).min()
    print(f"embeddings without the rotation: rel-L2 {moved:.3f}")
    assert moved > 50 * 1e-3


@pytest.mark.parametrize("style", ["hf", "trained"])
@pytest.mark.parametrize("pooling", ["mean", "cls"])
def test_emulated_floor_is_below_half_the_bar(style, pooling):
    """The whole forward with the kernels' fp16 operand and output roundings, against the fp64 oracle: the floor the GPU's
    1e-3 parity bar for 2-layer models must be at least twice.  (The golden generator records the same floor on its 12-layer
    and 8192-token cases; test_bars_are_at_least_twice_the_recorded_floors holds nomic_refs.BARS to it.)"""
    flat = N.make_weights(G2, 3, style)
    lens = [300, 77, 5]
    ids = _ids(np.random.default_rng(0), lens, 300)
    floor = _rel(N.emulate_forward(flat, ids, lens, G2, pooling), N.forward_np(flat, ids, lens, G2, pooling)).max()
    print(f"emulated fp16-operand floor ({style}, {pooling}, 2 layers): {floor:.2e}")
    assert floor < 0.5e-3


# ------------------------------------------------------------------------------------------------ weights and config

def _hf_state_dict(flat, g):
    sd = {"embeddings.word_embeddings.weight": flat["emb.word"], "embeddings.token_type_embeddings.weight": flat["emb.type"],
          "embeddings.LayerNorm.weight": flat["emb.ln.g"], "embeddings.LayerNorm.bias": flat["emb.ln.b"]}
    for l in range(g["layers"]):
        p, s = f"l{l}.", f"layers.{l}."
        q, k, v = np.split(flat[p + "qkv.w"], 3, 0)
        sd.update({s + "self_attn.q_proj.weight": q, s + "self_attn.k_proj.weight": k, s + "self_attn.v_proj.weight": v,
                   s + "self_attn.o_proj.weight": flat[p + "ao.w"], s + "post_attention_layernorm.weight": flat[p + "ln1.g"],
                   s + "post_attention_layernorm.bias": flat[p + "ln1.b"], s + "mlp.gate_proj.weight": flat[p + "gate.w"],
                   s + "mlp.up_proj.weight": flat[p + "up.w"], s + "mlp.down_proj.weight": flat[p + "down.w"],
                   s + "post_mlp_layernorm.weight": flat[p + "ln2.g"], s + "post_mlp_layernorm.bias": flat[p + "ln2.b"]})
    return sd


def _hub_state_dict(flat, g):
    """The hub checkpoint's (remote-code) names, as transformers' conversion mapping for "nomic_bert" lists them."""
    sd = {"embeddings.word_embeddings.weight": flat["emb.word"], "embeddings.token_type_embeddings.weight": flat["emb.type"],
          "emb_ln.weight": flat["emb.ln.g"], "emb_ln.bias": flat["emb.ln.b"]}
    for l in range(g["layers"]):
        p, s = f"l{l}.", f"encoder.layers.{l}."
        sd.update({s + "attn.Wqkv.weight": flat[p + "qkv.w"], s + "attn.out_proj.weight": flat[p + "ao.w"],
                   s + "norm1.weight": flat[p + "ln1.g"], s + "norm1.bias": flat[p + "ln1.b"], s + "mlp.fc12.weight": flat[p + "gate.w"],
                   s + "mlp.fc11.weight": flat[p + "up.w"], s + "mlp.fc2.weight": flat[p + "down.w"], s + "norm2.weight": flat[p + "ln2.g"],
                   s + "norm2.bias": flat[p + "ln2.b"]})
    return sd


def test_both_namings_load_to_the_same_blob():
    flat = N.make_weights(G2, 6, "trained")
    want = N.pack(flat, G2).view(np.uint32)
    for sd in (_hf_state_dict(flat, G2), _hub_state_dict(flat, G2), {"model." + k: v for k, v in _hf_state_dict(flat, G2).items()}):
        g, blob = W.load_hf_nomic_state_dict(sd, G2)
        assert (g["layers"], g["inter"], g["vocab"]) == (2, 3072, 30528)
        assert (blob.view(np.uint32) == want).all()


def test_the_hf_model_state_dict_loads():
    pytest.importorskip("transformers")
    flat = N.make_weights(G2, 6, "hf")
    sd = {k: v.numpy() for k, v in N.build_hf_model(flat, G2).state_dict().items()}
    _, blob = W.load_hf_nomic_state_dict(sd, G2)
    assert (blob.view(np.uint32) == N.pack(flat, G2).view(np.uint32)).all()


def test_a_projection_bias_is_refused():
    sd = _hub_state_dict(N.make_weights(G2, 6, "hf"), G2)
    sd["encoder.layers.0.attn.Wqkv.bias"] = np.zeros(2304, np.float32)
    with pytest.raises(ValueError, match="no bias"):
        W.load_hf_nomic_state_dict(sd, G2)


TRANSFORMERS_CONFIG = {"architectures": ["NomicBertModel"], "model_type": "nomic_bert", "vocab_size": 30528, "hidden_size": 768,
                       "num_attention_heads": 12, "intermediate_size": 3072, "num_hidden_layers": 12, "max_position_embeddings": 8192,
                       "layer_norm_eps": 1e-12, "rope_parameters": {"rope_type": "default", "rope_theta": 1000.0}}
# The remote-code config.json of nomic-ai/nomic-embed-text-v1.5 as remembered, not copied: nothing available offline confirms
# these field names or values.
REMOTE_CODE_CONFIG = {"architectures": ["NomicBertModel"], "model_type": "nomic_bert", "vocab_size": 30528, "n_embd": 768, "n_head": 12,
                      "n_inner": 3072, "n_layer": 12, "layer_norm_epsilon": 1e-12, "rotary_emb_base": 1000, "max_trained_positions": 2048,
                      "n_positions": 8192, "activation_function": "swiglu", "rotary_emb_fraction": 1.0, "rotary_emb_interleaved": False,
                      "prenorm": False, "qkv_proj_bias": False, "mlp_fc1_bias": False, "mlp_fc2_bias": False, "rotary_scaling_factor": None}


def test_config_reader():
    g = W.nomic_config(TRANSFORMERS_CONFIG)
    assert (g["hidden"], g["heads"], g["inter"], g["layers"], g["max_pos"], g["rope_theta"], g["eps"]) == (768, 12, 3072, 12, 8192, 1000.0, 1e-12)
    g = W.nomic_config(REMOTE_CODE_CONFIG)
    assert (g["hidden"], g["heads"], g["inter"], g["layers"], g["max_pos"], g["rope_theta"]) == (768, 12, 3072, 12, 2048, 1000.0)
    assert W.nomic_config({})["max_pos"] == 2048
    assert W.nomic_config(dict(TRANSFORMERS_CONFIG, max_position_embeddings=32768))["max_pos"] == 8192


@pytest.mark.parametrize("bad", [
    {"rope_parameters": {"rope_type": "yarn", "rope_theta": 1000.0}}, {"rotary_scaling_factor": 2.0}, {"rotary_emb_interleaved": True},
    {"rotary_emb_fraction": 0.5}, {"prenorm": True}, {"qkv_proj_bias": True}, {"mlp_fc1_bias": True}, {"activation_function": "gelu"},
])
def test_config_refusals(bad):
    with pytest.raises(ValueError):
        W.nomic_config(dict(REMOTE_CODE_CONFIG, **bad))


def test_is_nomic_dir(tmp_path):
    (tmp_path / "config.json").write_text(json.dumps(REMOTE_CODE_CONFIG))
    assert W.is_nomic_dir(str(tmp_path))
    (tmp_path / "config.json").write_text(json.dumps({"architectures": ["BertModel"], "model_type": "bert"}))
    assert not W.is_nomic_dir(str(tmp_path))


# ------------------------------------------------------------------------------------------------ kernel references and mutants

def _rope_case(M=192, S=64):
    rng = np.random.default_rng(2)
    a = (rng.standard_normal((M, 768)) * 1.2).astype(np.float16)
    w = (rng.standard_normal((2304, 768)) * 0.05).astype(np.float16)
    c = (rng.standard_normal(2304) * 0.1).astype(np.float32)
    v32 = (a.astype(np.float32) @ w.astype(np.float32).T + c).astype(np.float32)
    return a, w, c, v32, N.rope_table(4 * S, 1000.0), S


@pytest.mark.parametrize("mutant", [None, "interleaved", "pos_row", "sin_sign", "rotate_v", "pos_off"])
def test_rope_reference_rejects_mutants(mutant):
    a, w, c, v32, table, S = _rope_case()
    ref, tol = N.rope_gemm_ref(a, w, c, None, table, S, 1536, 1e-12)
    got = N.emulate_rope_epilogue(v32, table, S, 1536, mutant).astype(np.float64)
    if mutant is None:
        KR.check("rope emulation", got, ref, tol)
    else:
        with pytest.raises(AssertionError):
            KR.check(f"rope mutant {mutant}", got, ref, tol)


@pytest.mark.parametrize("mutant", [None, "swap", "gelu", "interleave4"])
def test_swiglu_reference_rejects_mutants(mutant):
    rng = np.random.default_rng(3)
    a = (rng.standard_normal((130, 768)) * 1.2).astype(np.float16)
    w = N.interleave_rows(rng.standard_normal((3072, 768)) * 0.05, rng.standard_normal((3072, 768)) * 0.05).astype(np.float16)
    c = (rng.standard_normal(6144) * 0.3).astype(np.float32)
    v32 = (a.astype(np.float32) @ w.astype(np.float32).T + c).astype(np.float32)
    ref, tol = N.swiglu_gemm_ref(a, w, c, None, 1e-12)
    got = N.emulate_swiglu_epilogue(v32, mutant).astype(np.float64)
    if mutant is None:
        KR.check("swiglu emulation", got, ref, tol)
    else:
        with pytest.raises(AssertionError):
            KR.check(f"swiglu mutant {mutant}", got, ref, tol)


@pytest.mark.parametrize("mutant", [None, "stale_stage", "unmasked_tail", "neighbour", "no_rescale", "half_keys"])
def test_streaming_attention_reference_rejects_mutants(mutant):
    """Keys that climb by 128-key tile (so a stage boundary raises the row max and a missing rescale shows), 1100 of 1152 valid
    (a partial last tile, 9 tiles: more than two laps of the 4-stage ring)."""
    B, S, lens = 2, 1152, [1100, 1100]
    qkv = N.synth_qkv(B, S, 5, q_scale=0.3).reshape(B, S, 3, 12, 64)
    qkv[:, :, 1] += (np.arange(S) // 128)[None, :, None, None].astype(np.float16) * np.float16(0.2) * qkv[:, :1, 0]
    qkv = qkv.reshape(B * S, 2304)
    rows = np.arange(0, S, 37)
    ref, tol = N.attention_rows_ref(qkv, lens, B, S, rows)
    got = N.emulate_attention_stream(qkv, lens, B, S, rows, mutant).astype(np.float64)
    if mutant is None:
        KR.check("attention_stream emulation", got, ref, tol)
    else:
        with pytest.raises(AssertionError):
            KR.check(f"attention_stream mutant {mutant}", got, ref, tol)


# ------------------------------------------------------------------------------------------------ router (host side)

class _FakeModel:
    """Stands in for the GPU model: records the ids it was given."""

    def __init__(self):
        self.calls = []

    def embed(self, ids, lens):
        self.calls.append((ids.copy(), lens.copy()))
        return np.zeros((len(ids), 768), np.float32)


def _engine(model_id, auto_truncate=False):
    from tei_router import server
    from tei_router.tokenizer import WordPiece

    args = server.parse_args(["--model-id", model_id] + (["--auto-truncate"] if auto_truncate else []))
    e = server.Engine.__new__(server.Engine)
    e.np, e.args, e.n_gpus, e.classifier, e.splade = np, args, 1, False, False
    e.pooling = server.resolve_pooling(None, None, model_id)
    e.tok = WordPiece(None)
    g, blob, source = server.load_weights(args)
    e.geometry, e.model = g, _FakeModel()
    return e, blob, source


def test_router_serves_nomic_ids_with_long_inputs():
    from tei_router import server

    for mid in server.NOMIC_MODEL_IDS:
        e, blob, source = _engine(mid)
        assert source is None and e.pooling == "mean"
        assert blob.size == sum(int(np.prod(s)) for _, s in W.nomic_blob_layout(e.geometry))
        info = e.info()
        assert info["max_input_length"] == 8192 and info["pooling"] == "mean"
        long_text = " ".join(["hello"] * 1000)
        n = len(e.tok.encode(long_text, 8192))
        assert 1500 < n <= 8192
        e.embed([long_text])
        assert e.model.calls[-1][1][0] == n  # past 512 and not truncated
        with pytest.raises(ValueError):  # TEI: 413
            e.embed([" ".join(["hello"] * 9000)])
        e.embed([" ".join(["hello"] * 9000)], truncate=True)
        assert e.model.calls[-1][1][0] == 8192
    # every other model's /info is as it was
    e, _, _ = _engine("BAAI/bge-base-en-v1.5")
    assert e.info()["max_input_length"] == 512


def serve(engine):
    """The router's HTTP handler around `engine` on an ephemeral port: (post(path, body) -> (status, json), get(path), stop)."""
    import threading
    import urllib.error
    import urllib.request
    from http.server import ThreadingHTTPServer

    from tei_router import server

    httpd = ThreadingHTTPServer(("127.0.0.1", 0), server.make_handler(engine))
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    base = f"http://127.0.0.1:{httpd.server_address[1]}"

    def call(path, body=None):
        req = urllib.request.Request(base + path, data=None if body is None else json.dumps(body).encode(),
                                     headers={"Content-Type": "application/json"})
        try:
            with urllib.request.urlopen(req, timeout=600) as r:
                return r.status, json.loads(r.read())
        except urllib.error.HTTPError as e:
            return e.code, json.loads(e.read())

    def stop():
        httpd.shutdown()
        httpd.server_close()

    return (lambda path, body: call(path, body)), (lambda path: call(path)), stop


def test_router_http_info_truncate_and_413():
    """Through the HTTP handler: /info's max_input_length, /embed past it answers 413, with "truncate": true it embeds the
    first 8192 tokens; a bge-base model's /embed keeps its answers (truncate is not honoured there, as before)."""
    e, _, _ = _engine("nomic-ai/nomic-embed-text-v1.5")
    post, get, stop = serve(e)
    try:
        code, info = get("/info")
        assert code == 200 and info["max_input_length"] == 8192
        long_text = " ".join(["hello"] * 9000)
        code, body = post("/embed", {"inputs": long_text})
        assert code == 413 and body["error_type"] == "Validation", body
        code, body = post("/embed", {"inputs": [long_text], "truncate": True})
        assert code == 200 and len(body) == 1 and len(body[0]) == 768
        assert e.model.calls[-1][1][0] == 8192
        code, body = post("/embed", {"inputs": "short text"})
        assert code == 200
    finally:
        stop()
    e, _, _ = _engine("BAAI/bge-base-en-v1.5")
    post, get, stop = serve(e)
    try:
        assert get("/info")[1]["max_input_length"] == 512
        code, _ = post("/embed", {"inputs": " ".join(["hello"] * 600), "truncate": True})
        assert code == 413
    finally:
        stop()


# ------------------------------------------------------------------------------------------------ HF golden

GOLDEN_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nomic_golden.npz")


def _golden_cases():
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_nomic_golden", os.path.join(os.path.dirname(GOLDEN_PATH), "make_nomic_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    return mg


def test_bars_are_at_least_twice_the_recorded_floors():
    """Each parity bar the GPU tests use (nomic_refs.BARS) against the emulated fp16-operand floors the golden generator
    recorded on its cases (12 layers up to 2048 tokens, 2 layers up to 8192)."""
    gold = np.load(GOLDEN_PATH)
    for name, (layers, _, style, _, lens) in _golden_cases().CASES.items():
        assert gold[f"{name}_lens"].tolist() == lens
        for pooling in ("mean", "cls"):
            floor = float(gold[f"{name}_floor_{pooling}"].max())
            bar = N.BARS[(layers, pooling)]
            print(f"{name} {pooling}: floor {floor:.2e}, bar {bar}")
            assert bar >= 2 * floor, (name, pooling, floor, bar)


def test_oracle_matches_the_hf_golden_at_8192_positions():
    """The fp64 oracle against the golden's HF fp32 vectors on the 2-layer 8k case's two shortest items (1000 and 513 tokens
    of a max_position_embeddings 8192 model) -- the longer items are checked on the GPU against the golden directly."""
    gold = np.load(GOLDEN_PATH)
    mg = _golden_cases()
    g, flat, ids, lens = mg.case_inputs("l2_trained_8k")
    assert (ids == gold["l2_trained_8k_ids"]).all()
    sel = [2, 3]
    hs = N.hidden_np(flat, ids[sel], lens[sel], g)
    for pooling in ("mean", "cls"):
        rel = _rel(gold[f"l2_trained_8k_{pooling}"][sel], N.pool(hs, pooling))
        assert rel.max() <= 5e-6, rel
