"""GPU (`-m gpu`): the second encoder on the same scheduler -- the CLIP ViT-B/16 image tower behind the reference's image
embedding example (06_gpu_and_ml/embeddings/image_embeddings_infinity.py:76-77, 298-306, 330-350) -- through the C ABI
(`b200rt_model_load("vit")`, `b200rt_submit_pixels`) against the oracle (oracle/clip_ref.py, pinned to HF
CLIPVisionModelWithProjection by tests/golden/clip_golden.npz).  Bars as for the text encoder: <= 1e-3 relative L2 per item;
random-weight image embeddings are strongly collinear (class token + positions dominate), so the item-specific part
(embedding minus the batch mean) is checked as well, at the tolerance its smaller norm implies."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import clip_ref as C

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_clip_golden", os.path.join(ROOT, "tests", "golden", "make_clip_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)


@pytest.fixture(scope="module")
def rt():
    import b200rt
    import torch

    b200rt.init(min(torch.cuda.device_count(), 8))
    yield b200rt
    b200rt.shutdown()


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "clip_golden.npz"))


_models = {}


def get_model(rt, layers, style, seed):
    key = (layers, style, seed)
    if key not in _models:
        g = C.VitGeometry(layers=layers)
        flat = C.make_weights(g, seed, style)
        _models[key] = (g, flat, rt.ImageEmbedModel(C.geometry_dict(g), C.pack_blob(flat, g)))
    return _models[key]


def test_residual_stream_layer_by_layer(rt):
    g, flat, model = get_model(rt, 2, "trained", 1)
    px = C.synth_pixels(3, g, 2)
    _, hidden = C.forward_np(flat, px, g, return_hidden=True)
    for L in range(g.layers + 1):
        got = model.debug_residual(px, L)
        rel = np.linalg.norm(got - hidden[L]) / np.linalg.norm(hidden[L])
        assert rel < (1e-3 if L else 6e-4), (L, rel)  # layer 0: fp16 pixels x fp16 patch weights, fp16 patch output, then pre_layrnorm


@pytest.mark.parametrize("case", ["VA", "VB", "VC"])
def test_image_embeddings_vs_golden(rt, golden, case):
    layers, style, wseed, n, pseed = mg.CASES[case]
    g, flat, model = get_model(rt, layers, style, wseed)
    px = C.synth_pixels(n, g, pseed)
    emb = model.embed(px)
    ref = golden[f"{case}_emb"]
    assert emb.shape == (n, g.proj) and np.allclose(np.linalg.norm(emb, axis=1), 1.0, atol=1e-5)
    rel = C.rel_l2(emb, ref)
    spec = C.rel_l2(emb - emb.mean(0), ref - ref.mean(0))
    print(f"case {case}: rel-L2 {rel.max():.3e}, item-specific part {spec.max():.3e} (its norm {np.linalg.norm(ref - ref.mean(0), axis=1).mean():.3f})")
    assert rel.max() <= 1e-3, rel
    assert spec.max() <= 3e-2, spec


def test_scheduler_waves_pool_and_text_model_side_by_side(rt):
    """More images than one wave holds, over every replica, interleaved with a text model on the same runtime: image and text
    tickets never share a wave and both come back right."""
    from oracle import bge_ref as R

    g, flat, model = get_model(rt, 2, "trained", 1)
    tg = R.BertGeometry(layers=2)
    tflat = R.make_weights(tg, 3, "trained")
    text = rt.EmbedModel(R.geometry_dict(tg), R.pack_blob(tflat, tg))
    n = 64 * rt.num_gpus() + 37
    px = np.tile(C.synth_pixels(8, g, 5), (n // 8 + 1, 1, 1, 1))[:n]
    ids = R.synth_ids(40, 128, 9)
    t_img = model.submit(px)
    t_txt = text.submit(ids)
    t_img2 = model.submit(px[:5])
    emb = model.wait(t_img, 120_000)
    first = model.embed(px[:8])
    for k in range(0, n - 8, 8):
        assert np.array_equal(emb[k:k + 8], first), k  # the same image gives the same bits wherever it travels
    assert np.array_equal(model.wait(t_img2, 60_000), first[:5])
    assert R.rel_l2(text.wait(t_txt, 60_000)[:3], R.forward_np(tflat, ids[:3], None, tg)).max() <= 1e-3
    assert C.rel_l2(first[:2], C.forward_np(flat, px[:2], g)).max() <= 1e-3
    import ctypes

    one = np.full((1, 8), 101, np.int32)
    o = np.zeros((1, 768), np.float32)
    t = ctypes.c_uint64(0)
    assert model._lib.b200rt_submit(model.handle, one.ctypes.data_as(ctypes.c_void_p), None, 1, 8, o.ctypes.data_as(ctypes.c_void_p), ctypes.byref(t)) == rt.E_INVALID
    with pytest.raises(rt.B200RTError):
        model.submit(np.zeros((1, 3, 32, 32), np.float32))


def test_second_image_size_is_refused_before_loading_weights(rt):
    """A second ViT with another image size is refused with E_UNSUPPORTED ahead of the blob-size check (E_INVALID), so before
    any of its weights are allocated on a replica; the loaded model embeds exactly as before."""
    import ctypes

    g, flat, model = get_model(rt, 2, "trained", 1)
    px = C.synth_pixels(2, g, 2)
    before = model.embed(px)
    cfg = rt.VitConfig(g.image // 2, g.patch, g.hidden, g.layers, g.heads, g.inter, g.proj, g.eps)
    wrong = np.zeros(16, np.float32)
    h = ctypes.c_int32(-1)
    assert model._lib.b200rt_model_load_ex(b"vit", ctypes.byref(cfg), rt._ptr(wrong), wrong.nbytes, 0, ctypes.byref(h)) == rt.E_UNSUPPORTED
    assert b"image size" in model._lib.b200rt_last_error()
    after = model.embed(px)
    assert np.array_equal(after, before)
    assert C.rel_l2(after, C.forward_np(flat, px, g)).max() <= 1e-3


def test_infinity_emb_adapter_matches_the_oracle_on_pil_images(rt, tmp_path):
    """The product's `infinity_emb` stand-in (what image_embeddings_infinity.py:296-306, 340-350 drives): engines started the
    reference's way -- several per process, one per concurrent input -- share one loaded model; PIL images go through
    preprocess.clip_preprocess and the sm_90a tower; vectors equal the oracle's on HF-CLIPImageProcessor pixels.  Weights
    come from a .safetensors checkpoint in HF CLIP naming (the real-checkpoint path)."""
    import asyncio

    from b200rt import weights as W
    from infinity_emb import AsyncEmbeddingEngine, EngineArgs
    from infinity_emb.primitives import Dtype, InferenceEngine
    from PIL import Image
    from transformers import CLIPImageProcessor

    g = C.VitGeometry(layers=2)
    flat = C.make_weights(g, 4, "trained")
    ckpt = str(tmp_path / "model.safetensors")
    W.write_safetensors(ckpt, C.flat_to_hf_state(flat, g))
    rng = np.random.default_rng(3)
    # smooth images (JPEG-like statistics); 224 x 224 as the reference's volume holds them, plus two that need resize + crop
    def img(h, w):
        base = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)
        return Image.fromarray(base).resize((w, h), Image.BICUBIC)

    images = [img(224, 224) for _ in range(9)] + [img(300, 400), img(512, 260)]
    args = EngineArgs(model_name_or_path="openai/clip-vit-base-patch16", batch_size=100, model_warmup=False, engine=InferenceEngine.torch,
                      dtype=Dtype.float16, device="cuda", weights=ckpt)

    async def run():
        engines = [AsyncEmbeddingEngine.from_args(args) for _ in range(4)]  # n_engines = max_concurrent_inputs (:283-306)
        for e in engines:
            await e.astart()
        outs = await asyncio.gather(*(e.image_embed(images=images) for e in engines))
        for e in engines:
            await e.astop()
        return outs

    outs = asyncio.run(run())
    assert rt.stats()["items"] > 0  # the fixture's runtime is still up: the adapter did not shut down a pool it does not own
    proc = CLIPImageProcessor(size={"shortest_edge": 224}, crop_size={"height": 224, "width": 224}, resample=3,
                              image_mean=[0.48145466, 0.4578275, 0.40821073], image_std=[0.26862954, 0.26130258, 0.27577711])
    px = proc(images=images, return_tensors="np")["pixel_values"].astype(np.float32)
    ref = C.forward_np(flat, px, g)
    first = np.stack(outs[0][0])
    assert outs[0][1] == len(images) and first.shape == (len(images), g.proj)
    for vecs, usage in outs[1:]:
        assert np.array_equal(np.stack(vecs), first)  # same bits from every engine object
    assert np.abs(np.linalg.norm(first, axis=1) - 1).max() < 1e-5
    assert C.rel_l2(first[:9], ref[:9]).max() <= 1e-3
    assert C.rel_l2(first[9:], ref[9:]).max() <= 3e-3  # resized inputs: PIL vs torchvision bicubic differ by <= 1 grey level
