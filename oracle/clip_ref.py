"""ORACLE (test infrastructure, not product): CPU restatement of the CLIP ViT-B/16 image tower behind the reference's image
embedding example -- ``06_gpu_and_ml/embeddings/image_embeddings_infinity.py:76-77`` (``openai/clip-vit-base-patch16``,
224 x 224 inputs) served by ``infinity_emb`` with ``engine=torch, dtype=float16`` (``:298-306``), whose image path is
``CLIPModel.get_image_features`` followed by L2 normalisation.  The arithmetic lives in Hugging Face
``transformers/models/clip/modeling_clip.py`` (un-vendored): ``CLIPVisionEmbeddings`` (patch conv, class token, positions),
``CLIPVisionTransformer`` (pre_layrnorm, pre-LN encoder layers with quick-GELU MLPs, post_layernorm on the class token) and
``CLIPVisionModelWithProjection.visual_projection``.

Only tests/, tools/, ``__graft_entry__.smoke()`` and bench.py may import this module.  Parity is unpinned by the reference
(it keeps no embedding value); the restatement is pinned against HF ``CLIPVisionModelWithProjection`` run here
(tests/golden/make_golden.py -> tests/golden/clip_golden.npz).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np


@dataclass(frozen=True)
class VitGeometry:
    """openai/clip-vit-base-patch16 vision tower."""

    image: int = 224
    patch: int = 16
    hidden: int = 768
    layers: int = 12
    heads: int = 12
    inter: int = 3072
    proj: int = 512
    eps: float = 1e-5

    @property
    def grid(self) -> int:
        return self.image // self.patch

    @property
    def tokens(self) -> int:
        return self.grid * self.grid + 1

    @property
    def patch_dim(self) -> int:
        return 3 * self.patch * self.patch


CLIP_B16 = VitGeometry()


def blob_layout(g: VitGeometry):
    """Flat fp32 blob both sides load.  HF shapes; the patch convolution weight [hidden, 3, p, p] is flattened to
    [hidden, 3*p*p] (channel, row, column order); q, k, v stacked to [3H, H]."""
    h, i = g.hidden, g.inter
    lay = [("patch.w", (h, g.patch_dim)), ("cls", (h,)), ("pos", (g.tokens, h)), ("pre.g", (h,)), ("pre.b", (h,))]
    for l in range(g.layers):
        p = f"l{l}."
        lay += [(p + "ln1.g", (h,)), (p + "ln1.b", (h,)), (p + "qkv.w", (3 * h, h)), (p + "qkv.b", (3 * h,)),
                (p + "ao.w", (h, h)), (p + "ao.b", (h,)), (p + "ln2.g", (h,)), (p + "ln2.b", (h,)),
                (p + "ff1.w", (i, h)), (p + "ff1.b", (i,)), (p + "ff2.w", (h, i)), (p + "ff2.b", (h,))]
    lay += [("post.g", (h,)), ("post.b", (h,)), ("proj.w", (g.proj, h))]
    return lay


def blob_numel(g: VitGeometry) -> int:
    return sum(int(np.prod(s)) for _, s in blob_layout(g))


def make_weights(g: VitGeometry = CLIP_B16, seed: int = 0, style: str = "hf") -> dict:
    """Seeded weights.  "hf": normal sigma 0.02 matrices/embeddings, zero biases, unit LayerNorm; "trained": non-zero biases
    and non-unit LayerNorm gains/offsets on top.

    "hard": the statistics of a trained pre-LN tower that seeded-normal weights never produce (drawn after the "hf" draws,
    so "hf" / "trained" keep their bits):
      * massive activations: three residual channels (HARD_CHANNELS) hold about 200 on the class token and, with the
        opposite signs, on two fixed patch tokens (HARD_PATCH_TOKENS), 60-125x the median |x| of the stream -- put there by the class
        embedding / the position rows and pre_layrnorm's gain on those channels.  The pre-LN stream is never renormalised,
        so they persist through every layer;
      * LN1 / LN2 / post_layernorm gains of 0.05 on those channels, and the columns that consume them (Q, V, FFN1, the
        projection) scaled down 25x;
      * an attention sink on the class token: in 8 of the 12 heads one query / key dimension reads only the massive channels
        (key) and a bias (query: 10 here, 6 in the text tower), so that 20-45 % of the (query, head) rows put more than half
        their weight on key 0;
      * peaked attention (Q and K 1.5x), LayerNorm gains around 2.5 (+-20 %), non-zero biases everywhere.
    Every activation stays far inside fp16 (below 2 000).  tests/test_gpu_pre_ln_chain.py asserts these statistics."""
    rng = np.random.default_rng(seed)
    flat = {}
    for name, shape in blob_layout(g):
        if name.endswith(".g"):
            flat[name] = np.ones(shape, np.float32)
        elif name.endswith(".b"):
            flat[name] = np.zeros(shape, np.float32)
        else:
            flat[name] = rng.standard_normal(shape, dtype=np.float32) * np.float32(0.02)
    if style == "trained":
        for name, shape in blob_layout(g):
            if name.endswith(".g"):
                flat[name] = (1.0 + 0.1 * rng.standard_normal(shape, dtype=np.float32)).astype(np.float32)
            elif name.endswith(".b"):
                flat[name] = (0.05 * rng.standard_normal(shape, dtype=np.float32)).astype(np.float32)
        for l in range(g.layers):
            flat[f"l{l}.qkv.w"][: 2 * g.hidden] *= np.float32(2.0)
    elif style == "hard":
        h = g.hidden
        pre_ln_hard(flat, blob_layout(g), h, g.heads, g.layers, "post.", rng, sink=10.0)
        ch = HARD_CHANNELS
        flat["pre.g"][ch] = np.float32(12.5)  # a row whose variance the three channels dominate: |z| ~ 16 there, x ~ 200
        flat["cls"][ch] = np.float32(20.0) * HARD_SIGNS
        for t in HARD_PATCH_TOKENS:
            flat["pos"][t, ch] = np.float32(-20.0) * HARD_SIGNS
        flat["patch.w"][ch] *= np.float32(0.05)  # ordinary patches stay ordinary on those channels
    elif style != "hf":
        raise ValueError(style)
    return flat


HARD_CHANNELS = np.array([37, 301, 470])  # the massive residual channels of the "hard" style (both CLIP towers)
HARD_SIGNS = np.array([1.0, -1.0, 1.0], np.float32)  # their signs on token 0
HARD_PATCH_TOKENS = (19, 150)  # ViT: two patch tokens that carry them too, with the opposite signs (no sink there)


def pre_ln_hard(flat: dict, layout, h: int, heads: int, layers: int, final: str, rng, sink: float) -> None:
    """The "hard" statistics both pre-LN CLIP towers share (see make_weights), drawn from `rng` after the "hf" draws: gains,
    biases, the scaled-down consumers of HARD_CHANNELS, peaked Q / K and the sink dimension of 2 heads in 3."""
    ch, hd = HARD_CHANNELS, h // heads
    for name, shape in layout:
        if name.endswith(".g"):
            gain = (2.5 * np.clip(1.0 + 0.2 * rng.standard_normal(shape, dtype=np.float32), 0.3, None)).astype(np.float32)
            gain[ch] = 0.05
            flat[name] = gain
        elif name.endswith(".b"):
            is_ln = name.endswith(("ln1.b", "ln2.b")) or name in ("pre.b", final + "b")
            off = ((0.1 if is_ln else 0.05) * rng.standard_normal(shape, dtype=np.float32)).astype(np.float32)
            if is_ln:
                off[ch] = 0.0
            flat[name] = off
    for l in range(layers):
        p = f"l{l}."
        w, b = flat[p + "qkv.w"], flat[p + "qkv.b"]
        w[: 2 * h] *= np.float32(1.5)
        w[:h, ch] *= np.float32(1.0 / 25.0)
        w[2 * h:, ch] *= np.float32(1.0 / 25.0)
        flat[p + "ff1.w"][:, ch] *= np.float32(1.0 / 25.0)
        for head in range(heads):
            if head % 3 == 2:
                continue
            j = head * hd + hd - 1  # the sink dimension: the key reads the massive channels only, the query a constant
            w[h + j] = 0.0
            w[h + j, ch] = np.float32(4.0) * HARD_SIGNS
            b[h + j] = 0.0
            w[j] *= np.float32(0.25)
            b[j] = np.float32(sink)
    flat["proj.w"][:, ch] *= np.float32(1.0 / 25.0)


def pack_blob(flat: dict, g: VitGeometry) -> np.ndarray:
    out = np.empty(blob_numel(g), np.float32)
    o = 0
    for name, shape in blob_layout(g):
        n = int(np.prod(shape))
        assert flat[name].shape == tuple(shape), (name, flat[name].shape, shape)
        out[o:o + n] = flat[name].reshape(-1)
        o += n
    return out


def geometry_dict(g: VitGeometry) -> dict:
    return dict(image=g.image, patch=g.patch, hidden=g.hidden, layers=g.layers, heads=g.heads, inter=g.inter, proj=g.proj, eps=g.eps)


def synth_pixels(n: int, g: VitGeometry = CLIP_B16, seed: int = 0) -> np.ndarray:
    """Already-preprocessed pixel_values [n, 3, image, image] fp32 (CLIP's processor output is roughly N(0, 1) per channel)."""
    return np.random.default_rng(seed).standard_normal((n, 3, g.image, g.image), dtype=np.float32)


def flat_to_hf_state(flat: dict, g: VitGeometry) -> dict:
    h = g.hidden
    sd = {
        "vision_model.embeddings.class_embedding": flat["cls"],
        "vision_model.embeddings.patch_embedding.weight": flat["patch.w"].reshape(h, 3, g.patch, g.patch),
        "vision_model.embeddings.position_embedding.weight": flat["pos"],
        "vision_model.pre_layrnorm.weight": flat["pre.g"], "vision_model.pre_layrnorm.bias": flat["pre.b"],
        "vision_model.post_layernorm.weight": flat["post.g"], "vision_model.post_layernorm.bias": flat["post.b"],
        "visual_projection.weight": flat["proj.w"],
    }
    for l in range(g.layers):
        s, p = f"vision_model.encoder.layers.{l}.", f"l{l}."
        for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
            sd[s + f"self_attn.{n}.weight"] = flat[p + "qkv.w"][j * h:(j + 1) * h]
            sd[s + f"self_attn.{n}.bias"] = flat[p + "qkv.b"][j * h:(j + 1) * h]
        sd[s + "self_attn.out_proj.weight"], sd[s + "self_attn.out_proj.bias"] = flat[p + "ao.w"], flat[p + "ao.b"]
        sd[s + "layer_norm1.weight"], sd[s + "layer_norm1.bias"] = flat[p + "ln1.g"], flat[p + "ln1.b"]
        sd[s + "layer_norm2.weight"], sd[s + "layer_norm2.bias"] = flat[p + "ln2.g"], flat[p + "ln2.b"]
        sd[s + "mlp.fc1.weight"], sd[s + "mlp.fc1.bias"] = flat[p + "ff1.w"], flat[p + "ff1.b"]
        sd[s + "mlp.fc2.weight"], sd[s + "mlp.fc2.bias"] = flat[p + "ff2.w"], flat[p + "ff2.b"]
    return sd


def _ln(x, gam, bet, eps):
    mu = x.mean(-1, keepdims=True)
    xc = x - mu
    return xc / np.sqrt((xc * xc).mean(-1, keepdims=True) + eps) * gam + bet


def forward_np(flat: dict, pixels: np.ndarray, g: VitGeometry = CLIP_B16, dtype=np.float64, return_hidden: bool = False):
    """L2-normalised image embeddings [n, proj] (modeling_clip.py: CLIPVisionEmbeddings.forward, CLIPEncoderLayer.forward
    -- pre-LN, quick_gelu = x * sigmoid(1.702 x) --, CLIPVisionTransformer.forward pooled = post_layernorm(h[:, 0]),
    CLIPVisionModelWithProjection.visual_projection; then x / ||x|| as infinity's image embedding does)."""
    W = {k: v.astype(dtype) for k, v in flat.items()}
    n = pixels.shape[0]
    h, nh, p, gr = g.hidden, g.heads, g.patch, g.grid
    dh = h // nh
    # stride-p convolution == GEMM over non-overlapping patches flattened (channel, row, column)
    patches = pixels.astype(dtype).reshape(n, 3, gr, p, gr, p).transpose(0, 2, 4, 1, 3, 5).reshape(n, gr * gr, 3 * p * p)
    x = np.concatenate([np.broadcast_to(W["cls"], (n, 1, h)), patches @ W["patch.w"].T], 1) + W["pos"][None]
    x = _ln(x, W["pre.g"], W["pre.b"], g.eps)
    hidden = [x.astype(np.float32)] if return_hidden else None
    T = g.tokens
    for l in range(g.layers):
        q_ = f"l{l}."
        y = _ln(x, W[q_ + "ln1.g"], W[q_ + "ln1.b"], g.eps)
        qkv = y @ W[q_ + "qkv.w"].T + W[q_ + "qkv.b"]
        q, k, v = (qkv[..., j * h:(j + 1) * h].reshape(n, T, nh, dh).transpose(0, 2, 1, 3) for j in range(3))
        s = (q @ k.transpose(0, 1, 3, 2)) / math.sqrt(dh)
        e = np.exp(s - s.max(-1, keepdims=True))
        ctx = ((e / e.sum(-1, keepdims=True)) @ v).transpose(0, 2, 1, 3).reshape(n, T, h)
        x = x + ctx @ W[q_ + "ao.w"].T + W[q_ + "ao.b"]
        y = _ln(x, W[q_ + "ln2.g"], W[q_ + "ln2.b"], g.eps)
        u = y @ W[q_ + "ff1.w"].T + W[q_ + "ff1.b"]
        u = u / (1.0 + np.exp(-1.702 * u))
        x = x + u @ W[q_ + "ff2.w"].T + W[q_ + "ff2.b"]
        if return_hidden:
            hidden.append(x.astype(np.float32))
    pooled = _ln(x[:, 0], W["post.g"], W["post.b"], g.eps)
    emb = pooled @ W["proj.w"].T
    emb = (emb / np.maximum(np.sqrt((emb * emb).sum(-1, keepdims=True)), 1e-12)).astype(np.float32)
    return (emb, hidden) if return_hidden else emb


def build_hf_model(flat: dict, g: VitGeometry = CLIP_B16):
    import torch
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    cfg = CLIPVisionConfig(hidden_size=g.hidden, intermediate_size=g.inter, num_hidden_layers=g.layers, num_attention_heads=g.heads,
                           image_size=g.image, patch_size=g.patch, projection_dim=g.proj, hidden_act="quick_gelu", layer_norm_eps=g.eps)
    m = CLIPVisionModelWithProjection(cfg).eval()
    sd = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in flat_to_hf_state(flat, g).items()}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


def forward_hf(model, pixels: np.ndarray) -> np.ndarray:
    import torch

    with torch.no_grad():
        e = model(pixel_values=torch.from_numpy(np.ascontiguousarray(pixels, dtype=np.float32))).image_embeds
        e = torch.nn.functional.normalize(e, p=2, dim=1)
    return e.numpy().astype(np.float32)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.sqrt(((a - b) ** 2).sum(-1)) / np.maximum(np.sqrt((b ** 2).sum(-1)), 1e-30)
