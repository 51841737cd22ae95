"""fp64 numpy restatement of the CLIP text tower (the text half of the reference's ``openai/clip-vit-base-patch16``,
image_embeddings_infinity.py:76-77, which infinity's ``embed(sentences=...)`` runs), an HF ``CLIPTextModelWithProjection``
wrapper, and a CPU emulation of the GPU path's fp16 rounding points (the parity floor).  Test infrastructure, like
oracle/clip_ref.py for the image tower; pinned against HF by tests/golden/clip_text_golden.npz.

The arithmetic restated is HF ``modeling_clip.py``: ``CLIPTextEmbeddings`` (token + position, no LayerNorm),
``CLIPEncoderLayer`` (pre-LN, causal self-attention with the padding mask, quick-GELU MLP), ``CLIPTextTransformer``
(final_layer_norm, pooled row chosen from the ids) and ``CLIPTextModelWithProjection.text_projection``; then x / ||x||.
"""
from __future__ import annotations

import math

import numpy as np

from b200rt.weights import CLIP_TEXT_B16_GEOMETRY, clip_text_blob_layout

BOS, EOS = 49406, 49407


def geometry(**kw) -> dict:
    g = dict(CLIP_TEXT_B16_GEOMETRY)
    g.update(kw)
    return g


def make_weights(g: dict, seed: int = 0, style: str = "hf") -> dict:
    """Seeded weights.  "hf": normal sigma 0.02 matrices/embeddings, zero biases, unit LayerNorm; "trained": non-zero biases,
    non-unit LayerNorm gains/offsets and sharper attention (Q, K rows doubled); "hard": oracle/clip_ref.make_weights' "hard"
    statistics for this tower -- the massive channels come from position row 0 (always <|startoftext|>, or the only token),
    +-200, and every query of the causal tower sees the sink on key 0."""
    rng = np.random.default_rng(seed)
    flat = {}
    for name, shape in clip_text_blob_layout(g):
        if name.endswith(".g"):
            flat[name] = np.ones(shape, np.float32)
        elif name.endswith(".b"):
            flat[name] = np.zeros(shape, np.float32)
        else:
            flat[name] = rng.standard_normal(shape, dtype=np.float32) * np.float32(0.02)
    if style == "trained":
        for name, shape in clip_text_blob_layout(g):
            if name.endswith(".g"):
                flat[name] = (1.0 + 0.1 * rng.standard_normal(shape, dtype=np.float32)).astype(np.float32)
            elif name.endswith(".b"):
                flat[name] = (0.05 * rng.standard_normal(shape, dtype=np.float32)).astype(np.float32)
        for l in range(g["layers"]):
            flat[f"l{l}.qkv.w"][: 2 * g["hidden"]] *= np.float32(2.0)
    elif style == "hard":
        from oracle import clip_ref as C

        C.pre_ln_hard(flat, clip_text_blob_layout(g), g["hidden"], g["heads"], g["layers"], "final.", rng, sink=6.0)
        flat["pos"][0, C.HARD_CHANNELS] = np.float32(200.0) * C.HARD_SIGNS  # position 0 (<|startoftext|>) carries them
    elif style != "hf":
        raise ValueError(style)
    return flat


def pack_blob(flat: dict, g: dict) -> np.ndarray:
    return np.concatenate([flat[n].reshape(-1) for n, _ in clip_text_blob_layout(g)]).astype(np.float32)


def flat_to_hf_state(flat: dict, g: dict, prefix: str = "text_model.") -> dict:
    h = g["hidden"]
    sd = {prefix + "embeddings.token_embedding.weight": flat["token"], prefix + "embeddings.position_embedding.weight": flat["pos"],
          prefix + "final_layer_norm.weight": flat["final.g"], prefix + "final_layer_norm.bias": flat["final.b"],
          "text_projection.weight": flat["proj.w"]}
    for l in range(g["layers"]):
        s, p = f"{prefix}encoder.layers.{l}.", f"l{l}."
        for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
            sd[s + f"self_attn.{n}.weight"] = flat[p + "qkv.w"][j * h:(j + 1) * h]
            sd[s + f"self_attn.{n}.bias"] = flat[p + "qkv.b"][j * h:(j + 1) * h]
        sd[s + "self_attn.out_proj.weight"], sd[s + "self_attn.out_proj.bias"] = flat[p + "ao.w"], flat[p + "ao.b"]
        sd[s + "layer_norm1.weight"], sd[s + "layer_norm1.bias"] = flat[p + "ln1.g"], flat[p + "ln1.b"]
        sd[s + "layer_norm2.weight"], sd[s + "layer_norm2.bias"] = flat[p + "ln2.g"], flat[p + "ln2.b"]
        sd[s + "mlp.fc1.weight"], sd[s + "mlp.fc1.bias"] = flat[p + "ff1.w"], flat[p + "ff1.b"]
        sd[s + "mlp.fc2.weight"], sd[s + "mlp.fc2.bias"] = flat[p + "ff2.w"], flat[p + "ff2.b"]
    return sd


def synth_ids(lens, S: int, seed: int, vocab: int = 49408, eos_pad: int = 0) -> np.ndarray:
    """[n, S] int32: <|startoftext|>, word ids in [1000, 49000), <|endoftext|> at len - 1 - eos_pad and, for eos_pad > 0,
    <|endoftext|> padding up to len - 1 (inside len); <|endoftext|> past len as the HF tokenizer pads."""
    rng = np.random.default_rng(seed)
    ids = np.full((len(lens), S), EOS, np.int32)
    for i, L in enumerate(lens):
        ids[i, :L] = rng.integers(1000, min(vocab, 49000), L)
        ids[i, 0] = BOS if L > 1 else ids[i, 0]
        if L > 1:
            ids[i, max(1, L - 1 - eos_pad):L] = EOS
    return ids


def pooled_positions(ids: np.ndarray, lens, eos_id: int) -> np.ndarray:
    """The row each item is pooled from, among its lens[i] valid ids: eos_id == 2 (HF's legacy branch) the first position of
    the largest id, else the first position equal to eos_id, 0 when there is none."""
    out = []
    for i, L in enumerate(lens):
        row = ids[i, :L]
        if eos_id == 2:
            out.append(int(np.argmax(row)))
        else:
            hit = np.nonzero(row == eos_id)[0]
            out.append(int(hit[0]) if hit.size else 0)
    return np.array(out)


def _ln(x, gam, bet, eps):
    mu = x.mean(-1, keepdims=True)
    xc = x - mu
    return xc / np.sqrt((xc * xc).mean(-1, keepdims=True) + eps) * gam + bet


def attention_np(q, k, v, lens, causal=True):
    """q, k, v [B, nh, S, dh] fp64; keys >= len and (causal) keys after the query masked."""
    B, nh, S, dh = q.shape
    s = (q @ k.transpose(0, 1, 3, 2)) / math.sqrt(dh)
    mask = np.arange(S)[None, :] >= np.asarray(lens)[:, None]
    mask = np.broadcast_to(mask[:, None, None, :], s.shape)
    if causal:
        mask = mask | (np.arange(S)[None, :] > np.arange(S)[:, None])[None, None]
    s = np.where(mask, -np.inf, s)
    e = np.exp(s - s.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)) @ v


def forward_np(flat: dict, ids: np.ndarray, lens, g: dict, dtype=np.float64, return_hidden: bool = False):
    """L2-normalised text embeddings [n, proj]; with return_hidden also the residual stream after 0..layers layers."""
    W = {k: v.astype(dtype) for k, v in flat.items()}
    n, S = ids.shape
    lens = np.asarray(lens if lens is not None else [S] * n)
    h, nh = g["hidden"], g["heads"]
    dh = h // nh
    x = W["token"][ids] + W["pos"][:S][None]
    hidden = [x.astype(np.float32)] if return_hidden else None
    for l in range(g["layers"]):
        p = f"l{l}."
        y = _ln(x, W[p + "ln1.g"], W[p + "ln1.b"], g["eps"])
        qkv = y @ W[p + "qkv.w"].T + W[p + "qkv.b"]
        q, k, v = (qkv[..., j * h:(j + 1) * h].reshape(n, S, nh, dh).transpose(0, 2, 1, 3) for j in range(3))
        ctx = attention_np(q, k, v, lens).transpose(0, 2, 1, 3).reshape(n, S, h)
        x = x + ctx @ W[p + "ao.w"].T + W[p + "ao.b"]
        y = _ln(x, W[p + "ln2.g"], W[p + "ln2.b"], g["eps"])
        u = y @ W[p + "ff1.w"].T + W[p + "ff1.b"]
        u = u / (1.0 + np.exp(-1.702 * u))
        x = x + u @ W[p + "ff2.w"].T + W[p + "ff2.b"]
        if return_hidden:
            hidden.append(x.astype(np.float32))
    pos = pooled_positions(ids, lens, g["eos_id"])
    pooled = _ln(x[np.arange(n), pos], W["final.g"], W["final.b"], g["eps"])
    emb = pooled @ W["proj.w"].T
    emb = (emb / np.maximum(np.sqrt((emb * emb).sum(-1, keepdims=True)), 1e-12)).astype(np.float32)
    return (emb, hidden) if return_hidden else emb


def build_hf_model(flat: dict, g: dict):
    import torch
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection

    cfg = CLIPTextConfig(vocab_size=g["vocab"], hidden_size=g["hidden"], intermediate_size=g["inter"], num_hidden_layers=g["layers"],
                         num_attention_heads=g["heads"], max_position_embeddings=g["max_pos"], projection_dim=g["proj"],
                         hidden_act="quick_gelu", layer_norm_eps=g["eps"], eos_token_id=g["eos_id"], bos_token_id=BOS, pad_token_id=1)
    cfg._attn_implementation = "eager"
    m = CLIPTextModelWithProjection(cfg).eval()
    sd = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in flat_to_hf_state(flat, g).items()}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


def forward_hf(model, ids: np.ndarray, lens) -> np.ndarray:
    import torch

    n, S = ids.shape
    mask = (np.arange(S)[None, :] < np.asarray(lens)[:, None]).astype(np.int64)
    with torch.no_grad():
        e = model(input_ids=torch.from_numpy(ids.astype(np.int64)), attention_mask=torch.from_numpy(mask)).text_embeds
        e = torch.nn.functional.normalize(e, p=2, dim=1)
    return e.numpy().astype(np.float32)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.sqrt(((a - b) ** 2).sum(-1)) / np.maximum(np.sqrt((b ** 2).sum(-1)), 1e-30)


# ------------------------------------------------------------------------ kernel references at kernel precision
def causal_attention_ref(qkv16, lens, B, S, heads=8, hd=64, rows=None):
    """What the causal attention kernel returns, in fp64 (keys >= len and keys after the query masked, len clamped to [1, S]),
    and its elementwise tolerance: tests/attention_refs.py's terms, per query row over the keys that row sees.  `rows`: for
    each item, the query rows (within the item, ascending) to compute; the result then holds those rows, item after item."""
    from kernel_refs import SUB16, U16, U32, acc_ulps

    qkv = np.asarray(qkv16, np.float16).reshape(B, S, 3, heads, hd)
    scale = 1.0 / np.sqrt(hd)
    out, tol = [], []
    for b in range(B):
        n = int(np.clip(lens[b], 1, S))
        x = qkv[b].astype(np.float64)
        qi = np.arange(S) if rows is None else np.asarray(rows[b], np.int64)
        q = (x[:, 0] if rows is None else x[qi, 0]).transpose(1, 0, 2)
        k, v = (x[:n, j].transpose(1, 0, 2) for j in (1, 2))
        s = q @ k.transpose(0, 2, 1)
        s_tol = acc_ulps(hd) * U32 * (np.abs(q) @ np.abs(k).transpose(0, 2, 1)) + 2.0 * U32 * np.abs(s)
        s = np.where(np.arange(n)[None, None, :] > qi[None, :, None], -np.inf, s)
        e = np.exp((s - s.max(-1, keepdims=True)) * scale)
        p = e / e.sum(-1, keepdims=True)
        ctx = p @ v
        pv = p @ np.abs(v)
        spread = pv + np.abs(ctx)
        t = (U16 * np.abs(ctx) + U16 * pv + SUB16 * p.max(-1, keepdims=True) * np.abs(v).sum(-2, keepdims=True)
             + scale * np.where(p > 0, s_tol, 0).max(-1, keepdims=True) * spread + (acc_ulps(n) + 16.0) * U32 * spread + SUB16)
        out.append(ctx.transpose(1, 0, 2).reshape(len(qi), -1))
        tol.append(t.transpose(1, 0, 2).reshape(len(qi), -1))
    return np.concatenate(out), np.concatenate(tol)


def check_causal_attention(what, ctx, qkv16, lens, B, S, rows=None):
    """`rows` as causal_attention_ref's: ctx then holds those query rows only, item after item."""
    import kernel_refs as KR

    ref, tol = causal_attention_ref(qkv16, lens, B, S, rows=rows)
    got = np.asarray(ctx, np.float16).astype(np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output (padded query rows must stay finite too)"
    return KR.check(what, got, ref, tol)


def clip_text_pool_ref(hi, lo, ids, lens, gamma, beta, proj, S, eps, eos_id):
    """What clip_text_pool_kernel returns, in fp64 (the pooled row of each item, final LayerNorm, projection, L2 normalise),
    and its tolerance (kernel_refs.vit_pool_ref's terms at width 512)."""
    import kernel_refs as KR

    n = np.asarray(hi).shape[0] // S
    L = np.clip(np.asarray(lens), 1, S)
    pos = pooled_positions(np.asarray(ids).reshape(n, S), L, eos_id)
    rows = KR.hilo64(hi, lo).reshape(n, S, -1)[np.arange(n), pos]
    z, z_tol, _ = KR.layernorm_ref(rows, gamma, beta, eps)
    w = np.asarray(proj, np.float32).astype(np.float64)
    y_tol = z_tol @ np.abs(w).T + 30.0 * KR.U32 * (np.abs(z) @ np.abs(w).T)
    return KR._normalised(z @ w.T, y_tol, 8 + KR.LN_SUM_ULPS)


def check_clip_text_pool(what, out, hi, lo, ids, lens, gamma, beta, proj, S, eps, eos_id):
    import kernel_refs as KR

    ref, tol = clip_text_pool_ref(hi, lo, ids, lens, gamma, beta, proj, S, eps, eos_id)
    return KR.check(what, out, ref, tol)


# ------------------------------------------------------------------------ fp16-operand floor (CPU emulation of the GPU path)
def emulate(flat: dict, ids: np.ndarray, lens, g: dict) -> np.ndarray:
    """The GPU path's rounding points on the CPU: the residual stream kept in fp32 (hi + lo), fp16(y) against fp16 weights with
    LN1 / LN2 folded into the columns (rows centred), fp16 QKV, fp16 P, fp16 ctx, fp16 FFN activations, fp32 accumulation."""
    f16 = lambda a: a.astype(np.float16).astype(np.float32)  # noqa: E731
    W = {k: v.astype(np.float32) for k, v in flat.items()}
    n, S = ids.shape
    lens = np.asarray(lens)
    h, nh = g["hidden"], g["heads"]
    dh = h // nh
    y = W["token"][ids] + W["pos"][:S][None]

    def stats(y):
        mu = y.mean(-1, keepdims=True, dtype=np.float32)
        xc = y - mu
        return (1.0 / np.sqrt((xc * xc).mean(-1, keepdims=True, dtype=np.float32) + g["eps"])).astype(np.float32)

    def folded(y, lg, lb, w, b):
        wg = W[w] * W[lg][None, :]
        wp = f16(wg - wg.mean(1, keepdims=True, dtype=np.float32))
        return stats(y) * (f16(y) @ wp.T) + (W[w] @ W[lb] + W[b])

    mask = (np.arange(S)[None, :] >= lens[:, None])[:, None, None, :] | (np.arange(S)[None, :] > np.arange(S)[:, None])[None, None]
    for l in range(g["layers"]):
        p = f"l{l}."
        qkv = f16(folded(y, p + "ln1.g", p + "ln1.b", p + "qkv.w", p + "qkv.b"))
        q, k, v = (qkv[..., j * h:(j + 1) * h].reshape(n, S, nh, dh).transpose(0, 2, 1, 3) for j in range(3))
        s = np.where(mask, -np.inf, q @ k.transpose(0, 1, 3, 2))
        e = np.exp2((s - s.max(-1, keepdims=True)) * np.float32(1.4426950408889634 / math.sqrt(dh))).astype(np.float32)
        ctx = f16((f16(e) @ v) / e.sum(-1, keepdims=True, dtype=np.float32)).transpose(0, 2, 1, 3).reshape(n, S, h)
        y = y + (ctx @ f16(W[p + "ao.w"]).T + W[p + "ao.b"])
        u = folded(y, p + "ln2.g", p + "ln2.b", p + "ff1.w", p + "ff1.b")
        u = f16(u / (1.0 + np.exp(-1.702 * u)))
        y = y + (u @ f16(W[p + "ff2.w"]).T + W[p + "ff2.b"])
    pos = pooled_positions(ids, lens, g["eos_id"])
    pooled = _ln(y[np.arange(n), pos].astype(np.float64), W["final.g"], W["final.b"], g["eps"]).astype(np.float32)
    emb = pooled @ W["proj.w"].T
    return emb / np.maximum(np.sqrt((emb * emb).sum(-1, keepdims=True)), 1e-12)
