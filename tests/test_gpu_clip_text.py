"""GPU (`-m gpu`): the CLIP text tower (kind "clip_text") -- causal 8-head attention, the 512-wide GEMM epilogues and row
kernels, every launch of the forward against its kernel reference (ClipTextChain, through tests/test_gpu_forward_chain.py's
run_chain), golden parity, batch / replica invariance, a mixed runtime, the refusals and the
infinity_emb adapter end to end.

Parity bar: 2e-3 relative L2 per item.  The tower's fp16-operand floor, emulated on the CPU (clip_text_refs.emulate: fp16
GEMM operands, fp16 QKV / P / ctx / FFN activations, fp32 accumulation, the residual in fp32), is up to 8.8e-4 on the golden
cases (TB, 12 layers, 77 tokens), which leaves no margin under 1e-3."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

import clip_text_refs as T
import kernel_refs as KR
import test_gpu_forward_chain as FC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_clip_text_golden", os.path.join(ROOT, "tests", "golden", "make_clip_text_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)
BAR = 2e-3  # floor 8.8e-4 (see the module docstring)


@pytest.fixture(scope="module")
def rt():
    import b200rt
    import torch

    b200rt.init(min(torch.cuda.device_count(), 8))
    yield b200rt
    b200rt.shutdown()


_models = {}


def get_model(rt, layers, style, seed, eos_id=2):
    key = (layers, style, seed, eos_id)
    if key not in _models:
        g = T.geometry(layers=layers, eos_id=eos_id)
        flat = T.make_weights(g, seed, style)
        _models[key] = (g, flat, rt.ClipTextModel(g, T.pack_blob(flat, g)))
    return _models[key]


# ------------------------------------------------------------------------------------------------ causal attention
@pytest.mark.parametrize("S", [64, 128, 192, 512])
def test_causal_attention_vs_fp64(rt, S):
    lens = sorted({1, 2, 37, S} | {x for x in (64, 65, 127, 128, 129, 191, 192, 255, 256, 257, 383, 511) if x <= S})
    B = len(lens)
    rng = np.random.default_rng(S)
    qkv = (rng.standard_normal((B * S, 3 * 512)) * 1.5).astype(np.float16)
    ctx, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S, head_dim=64, heads=8, causal=True)
    T.check_causal_attention(f"causal attention S={S}", ctx, qkv, lens, B, S)
    one, _ = rt.debug_attention(qkv, np.array(lens, np.int32), B, S, head_dim=64, heads=8, causal=True, sms=1)
    assert np.array_equal(one.view(np.uint16), ctx.view(np.uint16))  # sms = 1 walks every unit on one CTA
    # query-tile split (a lone item spreads over 4 x 8 units when it has fewer units than SMs) vs the batch of all items
    for i in (0, B - 1):
        alone, _ = rt.debug_attention(qkv[i * S:(i + 1) * S], np.array([lens[i]], np.int32), 1, S, head_dim=64, heads=8, causal=True)
        assert np.array_equal(alone.view(np.uint16), ctx[i * S:(i + 1) * S].view(np.uint16)), i
    # masked keys carry exactly zero weight: change every future / padding key and value, the output keeps its bits
    q2 = qkv.copy().reshape(B, S, 3, 512)
    L = lens[-1]
    q2[-1, L // 2:, 1:] = np.float16(7.0)
    c2, _ = rt.debug_attention(q2.reshape(B * S, -1), np.array(lens, np.int32), B, S, head_dim=64, heads=8, causal=True)
    assert np.array_equal(c2[(B - 1) * S:(B - 1) * S + L // 2].view(np.uint16), ctx[(B - 1) * S:(B - 1) * S + L // 2].view(np.uint16))


# ------------------------------------------------------------------------------------------------ GEMM at width 512
def test_plain_debug_gemm_keeps_refusing_a_512_wide_layernorm(rt):
    a = np.zeros((64, 512), np.float16)
    with pytest.raises(rt.B200RTError) as e:
        rt.debug_gemm(0, a, np.zeros((512, 512), np.float16), np.zeros(512, np.float32), ln_stats=np.zeros((64, 4, 2), np.float32))
    assert e.value.code == rt.E_INVALID


LN512_CASES = ((0, 1536), (3, 2048))  # (epi, N): the tower's QKV and quick-GELU FFN1, K = 512 (4 partials)


@pytest.mark.parametrize("M", [1, 127, 128, 129, 300])
def test_gemm_512_wide_layernorm_epilogues(rt, M):
    rng = np.random.default_rng(M)
    y = (rng.standard_normal((M, 512)) * 3 + 0.5).astype(np.float32)
    st = KR.partials(y.astype(np.float64)).astype(np.float32)
    a16 = y.astype(np.float16)
    for epi, N in LN512_CASES:
        w = (rng.standard_normal((N, 512)) * 0.03).astype(np.float32)
        w16 = (w - w.mean(1, keepdims=True)).astype(np.float16)
        bias = (rng.standard_normal(N) * 0.1).astype(np.float32)
        out, _ = rt.debug_gemm(epi, a16, w16, bias, ln_stats=st, eps=1e-5, ln512=True)
        KR.check_gemm(f"epi {epi} M={M} K=512 4 partials", out.astype(np.float64), epi, a16, w16, bias, ln_stats=st, eps=1e-5)
    # pre-LN residual at N = 512: stats_in NULL, 4 partials per row emitted (two 256-column tiles, two each)
    for K in (512, 2048):
        a = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
        w16 = (rng.standard_normal((512, K)) * 0.03).astype(np.float16)
        bias = (rng.standard_normal(512) * 0.1).astype(np.float32)
        resid = (rng.standard_normal((M, 512)) * 2).astype(np.float32)
        out, _, so = rt.debug_gemm(2, a, w16, bias, resid=resid, want_stats=True)
        KR.check_gemm(f"epi 2 M={M} N=512 K={K}", out, 2, a, w16, bias, resid=resid)
        assert so.shape == (M, 4, 2)
        KR.check_gemm_stats(f"epi 2 partials M={M} K={K}", so, (a, w16, bias), resid=resid)


# ------------------------------------------------------------------------------------------------ row kernels
def test_embed_512_with_zero_type_row_is_token_plus_position(rt):
    rng = np.random.default_rng(1)
    word = rng.standard_normal((1000, 512)).astype(np.float32)
    pos = rng.standard_normal((128, 512)).astype(np.float32)
    S = 128
    ids = rng.integers(0, 1000, 3 * S).astype(np.int32)
    hi, lo, st = rt.debug_embed(ids, word, pos, np.zeros(512, np.float32), S, hidden=512)
    x = word[ids] + pos[np.arange(ids.size) % S]  # CLIPTextEmbeddings: token + position, no LayerNorm
    want_hi = x.astype(np.float16)
    KR.check_bits("embed 512 hi", hi, want_hi)
    KR.check_bits("embed 512 lo", lo, (x - want_hi.astype(np.float32)).astype(np.float16))
    KR.check_partials("embed 512 partials", st, x.astype(np.float64))


def test_clip_text_pool_vs_fp64(rt):
    rng = np.random.default_rng(2)
    S, n = 128, 6
    x = (rng.standard_normal((n * S, 512)) * 2).astype(np.float32)
    hi, lo = KR.split_hilo(x)
    g = (1 + 0.1 * rng.standard_normal(512)).astype(np.float32)
    b = (0.05 * rng.standard_normal(512)).astype(np.float32)
    proj = (rng.standard_normal((512, 512)) * 0.04).astype(np.float32)
    lens = np.array([77, 40, 30, 1, 10, 50], np.int32)
    ids = rng.integers(1000, 40000, (n, S)).astype(np.int32)
    ids[0, 0], ids[0, 76] = T.BOS, T.EOS                      # EOS at len - 1
    ids[1, 0], ids[1, 20:40] = T.BOS, T.EOS                   # 49407 padding after EOS inside len
    ids[2, :] = np.arange(S) % 37 + 100                       # no EOS: largest id at 36 / row 0 for first-match
    ids[3, 0] = 5                                              # len = 1
    ids[4, 10:] = 49407                                        # large ids past len are never read
    ids[5, :] = -7                                             # unvalidated device ids, all negative: row 0, never out of range
    for eos in (2, 49407):
        out = rt.debug_clip_text_pool(hi, lo, ids, lens, g, b, proj, S, 1e-5, eos)
        pos = T.pooled_positions(ids, lens, eos)
        T.check_clip_text_pool(f"clip_text_pool eos_id={eos} positions {pos.tolist()}", out, hi, lo, ids, lens, g, b, proj, S, 1e-5, eos)


# ------------------------------------------------------------------------------------------------ the forward
class ClipTextChain:
    """The text tower's weights as the engine holds them (pre-LN as tests/test_gpu_forward_chain.py's VitChain: LN1 folded
    into QKV, LN2 into FFN1, no LayerNorm re-applied to the residual), the batch, and the check of each launch at its kernel
    reference's precision on the operands the launch consumed.  The embedding reads the position table as the engine pads it
    (128 rows, zero past max_pos).  `rows` as tests/test_gpu_forward_chain.py's TextChain."""

    def __init__(self, flat, g, ids, lens, fold, rows=None):
        self.flat, self.g = flat, g
        self.ids, self.lens = np.asarray(ids, np.int32), np.asarray(lens, np.int32)
        self.B, self.S = self.ids.shape
        self.M = self.B * self.S
        FC.set_rows(self, rows)
        f, L, H = flat, g["layers"], g["hidden"]
        self.pos = np.zeros((128, H), np.float32)
        self.pos[:g["max_pos"]] = f["pos"]
        self.qkv = [fold(f[f"l{l}.qkv.w"], f[f"l{l}.ln1.g"], f[f"l{l}.ln1.b"], f[f"l{l}.qkv.b"]) for l in range(L)]
        self.ff1 = [fold(f[f"l{l}.ff1.w"], f[f"l{l}.ln2.g"], f[f"l{l}.ln2.b"], f[f"l{l}.ff1.b"]) for l in range(L)]
        self.ao16 = [fold(f[f"l{l}.ao.w"])[0] for l in range(L)]
        self.ff216 = [fold(f[f"l{l}.ff2.w"])[0] for l in range(L)]

    def check(self, tag, name, l, prev, cur):
        M, g, f, p, S = self.M, self.g, self.flat, f"l{l}.", self.S
        eps = g["eps"]
        P = lambda t, b: t[b][self.rows]  # noqa: E731
        A = lambda t, b: t[b][:M]  # noqa: E731
        what = f"{tag} layer {l} {name}"
        if name == "embed":
            return KR.check_embed(what, A(cur, "yhi"), A(cur, "ylo"), P(cur, "pstats0"), self.ids.reshape(-1), f["token"], self.pos[:S],
                                  np.zeros(g["hidden"], np.float32), S, rows=self.rows)
        if name == "gemm_qkv":
            w16, c = self.qkv[l]
            return KR.check_gemm(what, P(cur, "qkv"), 0, P(prev, "yhi"), w16, c, ln_stats=P(prev, "pstats0"), eps=eps)
        if name == "attention":
            return T.check_causal_attention(what, P(cur, "ctx"), A(prev, "qkv"), self.lens, self.B, S, rows=self.q_rows)
        if name == "gemm_attn_out":
            return FC._check_residual(what, cur, "pstats1", self.rows, (P(prev, "ctx"), self.ao16[l], f[p + "ao.b"]),
                                      dict(resid_hilo=(P(prev, "yhi"), P(prev, "ylo"))))
        if name == "gemm_ffn1_qgelu":
            w16, c = self.ff1[l]
            return KR.check_gemm(what, P(cur, "ffn"), 3, P(prev, "yhi"), w16, c, ln_stats=P(prev, "pstats1"), eps=eps)
        if name == "gemm_ffn2":
            return FC._check_residual(what, cur, "pstats0", self.rows, (P(prev, "ffn"), self.ff216[l], f[p + "ff2.b"]),
                                      dict(resid_hilo=(P(prev, "yhi"), P(prev, "ylo"))))
        if name == "clip_text_pool":
            return T.check_clip_text_pool(what, cur["out"], A(prev, "yhi"), A(prev, "ylo"), self.ids, self.lens, f["final.g"], f["final.b"],
                                          f["proj.w"], S, eps, g["eos_id"])
        raise AssertionError(f"{tag}: unexpected launch {name!r}")


@pytest.mark.parametrize("eos_id", [2, 49407])
def test_clip_text_chain(rt, eos_id):
    """Every launch of a 2-layer tower through tests/test_gpu_forward_chain.py's run_chain (its buffer invariants: nothing
    written past M, guard rows still poison, every row < M finite, padding included) on a ragged batch in the 128-token
    bucket -- items of 65-77 tokens travel there, so the embedding reads position rows 77-127 of the padded table for the
    padding rows.  Then the product path: embed() of the same items, through the scheduler's 64- and 128-token buckets and
    graph replay, is bitwise the traced pooled output, and one forward is 5 L + 2 launches (+ the wave's scatter)."""
    g, flat, model = get_model(rt, 2, "trained", 1, eos_id)
    lens = np.array([77, 1, 64, 65, 30, 2], np.int32)
    ids = T.synth_ids(lens, 128, seed=5)  # <|endoftext|> padding past len, as the tokenizer pads
    ids[4, 10:14] = T.EOS                 # an end token inside len before the last one
    ch = ClipTextChain(flat, g, ids, lens, FC.gpu_fold(rt))
    margins = {}
    last = FC.run_chain(f"clip_text eos {eos_id}", ch, lambda k: model.debug_trace(ids, lens, k), margins)
    FC.print_margins(f"clip_text eos {eos_id}", margins)
    assert last["n_total"] == 5 * g["layers"] + 2 and last["names"][0] == "embed"
    e = model.embed(ids[:, :77], lens)
    assert np.array_equal(e.view(np.uint32), last["out"].view(np.uint32)), "embed() differs from the traced pooled output"
    n0 = rt.stats()["kernel_launches"]
    model.embed(ids[:1, :77], lens[:1])
    assert rt.stats()["kernel_launches"] - n0 == last["n_total"] + 1
    _, _, m12 = get_model(rt, 12, "hf", 0)
    assert m12.debug_trace(ids, lens, 0)["n_total"] == 62


@pytest.mark.parametrize("case", list(mg.CASES))
def test_golden_parity(rt, case):
    golden = np.load(os.path.join(ROOT, "tests", "golden", "clip_text_golden.npz"))
    layers, style, seed, eos, _, _ = mg.CASES[case]
    g, flat, model = get_model(rt, layers, style, seed, eos)
    emb = model.embed(golden[f"{case}_ids"], golden[f"{case}_lens"])
    rel = T.rel_l2(emb, golden[f"{case}_emb"])
    print(f"case {case}: rel-L2 vs HF fp32 {rel.max():.3e} (bar {BAR:g}, fp16 floor <= 8.8e-4)")
    assert emb.shape == (len(golden[f"{case}_lens"]), 512) and np.allclose(np.linalg.norm(emb, axis=1), 1, atol=1e-5)
    assert rel.max() <= BAR, rel


def test_item_is_bitwise_the_same_alone_in_a_full_wave_and_on_every_replica(rt):
    g, flat, model = get_model(rt, 2, "trained", 1)
    n = 528
    rng = np.random.default_rng(7)
    lens = rng.integers(2, 78, n).astype(np.int32)
    ids = T.synth_ids(lens, 77, seed=8)
    full = model.embed(ids, lens)
    for i in (0, 1, 263, n - 1):
        alone = model.embed(ids[i:i + 1, :lens[i]], lens[i:i + 1])
        assert np.array_equal(alone, full[i:i + 1]), i
    # every replica (a small wave rotates its first replica)
    for _ in range(rt.num_gpus()):
        assert np.array_equal(model.embed(ids[:3], lens[:3]), full[:3])


def test_mixed_runtime_text_image_and_bge(rt):
    from oracle import bge_ref as R
    from oracle import clip_ref as C

    g, flat, model = get_model(rt, 2, "trained", 1)
    vg = C.VitGeometry(layers=2)
    img = rt.ImageEmbedModel(C.geometry_dict(vg), C.pack_blob(C.make_weights(vg, 1, "trained"), vg))
    bg = R.BertGeometry(layers=2)
    bge = rt.EmbedModel(R.geometry_dict(bg), R.pack_blob(R.make_weights(bg, 3, "trained"), bg))
    ids, lens = T.synth_ids([9, 77, 30], 77, seed=1), np.array([9, 77, 30], np.int32)
    px = C.synth_pixels(3, vg, 4)
    bids = R.synth_ids(4, 96, 2)
    alone = (model.embed(ids, lens), img.embed(px), bge.embed(bids))
    tickets = [model.submit(ids, lens), img.submit(px), bge.submit(bids), model.submit(ids, lens), img.submit(px)]
    got = [m.wait(t, 60_000) for m, t in zip((model, img, bge, model, img), tickets)]
    for a, b in zip(got, (alone[0], alone[1], alone[2], alone[0], alone[1])):
        assert np.array_equal(a, b)


def test_refusals(rt):
    lib = rt.load_library()
    g = dict(T.geometry(layers=1), hidden=768, heads=12, inter=3072)
    with pytest.raises(rt.B200RTError) as e:
        rt.ClipTextModel(g, np.zeros(10, np.float32))
    assert e.value.code == rt.E_UNSUPPORTED
    _, _, model = get_model(rt, 2, "trained", 1)
    with pytest.raises(rt.B200RTError) as e:
        model.embed(np.full((1, 78), 320, np.int32))
    assert e.value.code == rt.E_INVALID
    with pytest.raises(rt.B200RTError) as e:
        model.embed(np.array([[49406, 49408, 49407]], np.int32))
    assert e.value.code == rt.E_INVALID
    out = np.zeros((1, 512), np.float32)
    t = ctypes.c_uint64(0)
    px = np.zeros((1, 3, 224, 224), np.float32)
    assert lib.b200rt_submit_pixels(model.handle, px.ctypes.data_as(ctypes.c_void_p), 1, out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(t)) == rt.E_INVALID
    gs = T.geometry(layers=1, vocab=1000)
    blob = T.pack_blob(T.make_weights(gs, 0), gs)
    cfg = rt.ClipTextConfig(*(gs[k] for k in ("vocab", "hidden", "layers", "heads", "inter", "max_pos", "proj", "eos_id", "eps")))
    h = ctypes.c_int32(-1)
    assert lib.b200rt_model_load_ex(b"clip_text", ctypes.byref(cfg), blob.ctypes.data_as(ctypes.c_void_p), blob.nbytes, 1, ctypes.byref(h)) == rt.E_INVALID


def test_infinity_emb_adapter_text_and_image_search(rt, tmp_path):
    """Both towers of one seeded CLIPModel checkpoint through the infinity_emb stand-in: `embed(sentences=...)` equals the
    oracle on the same token ids, and 100 cos(image, text) is HF CLIPModel's logits_per_image."""
    import asyncio
    import json

    import torch
    from b200rt import weights as W
    from infinity_emb import AsyncEmbeddingEngine, EngineArgs
    from infinity_emb.clip_tokenizer import ClipTokenizer
    from oracle import clip_ref as C
    from transformers import CLIPConfig, CLIPModel

    vg = C.VitGeometry(layers=2)
    vflat = C.make_weights(vg, 4, "trained")
    tg = T.geometry(layers=2)
    tflat = T.make_weights(tg, 6, "trained")
    sd = dict(C.flat_to_hf_state(vflat, vg), **T.flat_to_hf_state(tflat, tg), logit_scale=np.array(np.log(100.0), np.float32))
    W.write_safetensors(str(tmp_path / "model.safetensors"), sd)
    json.dump({"text_config": {"eos_token_id": 2}}, open(tmp_path / "config.json", "w"))
    texts = ["a photo of a cat", "a diagram", "two dogs playing in the snow on a sunny day"]
    px = C.synth_pixels(2, vg, 9)
    args = EngineArgs(model_name_or_path=str(tmp_path))

    async def run():
        engines = [AsyncEmbeddingEngine.from_args(args) for _ in range(2)]
        for e in engines:
            await e.astart()
        t = await asyncio.gather(*(e.embed(sentences=texts) for e in engines))
        for e in engines:
            await e.astop()
        return t

    outs = asyncio.run(run())
    vecs, usage = outs[0]
    assert np.array_equal(np.stack(outs[1][0]), np.stack(vecs))
    tok = ClipTokenizer.from_dir(None)  # no vocab.json in the snapshot: the base vocabulary
    ids, lens = tok.batch(texts)
    assert usage == int(lens.sum())
    got = np.stack(vecs)
    assert T.rel_l2(got, T.forward_np(tflat, ids, lens, tg)).max() <= BAR
    img = np.stack([rt.ImageEmbedModel(C.geometry_dict(vg), C.pack_blob(vflat, vg)).embed(px)])[0]
    cfg = CLIPConfig(text_config=dict(vocab_size=49408, hidden_size=512, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=8,
                                      max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5, eos_token_id=2),
                     vision_config=dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12, image_size=224,
                                        patch_size=16, hidden_act="quick_gelu", layer_norm_eps=1e-5), projection_dim=512)
    hf = CLIPModel(cfg).eval()
    hf.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=False)
    with torch.no_grad():
        mask = (np.arange(ids.shape[1])[None, :] < lens[:, None]).astype(np.int64)
        logits = hf(input_ids=torch.from_numpy(ids.astype(np.int64)), attention_mask=torch.from_numpy(mask),
                    pixel_values=torch.from_numpy(px)).logits_per_image.numpy()
    ours = 100.0 * img @ got.T
    print("logits_per_image", logits.tolist(), "ours", ours.tolist())
    assert np.abs(ours - logits).max() <= 100.0 * 2 * BAR
