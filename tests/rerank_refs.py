"""fp64 oracle of BERT sequence classifiers (cross-encoders such as cross-encoder/ms-marco-MiniLM-L-6-v2, HF
``BertForSequenceClassification``), the kernel references of what the classifier path adds (embed with token types, the
pooler / classifier head), and numpy emulations of those kernels with the mutants their checks must reject.

The encoder is oracle/bge_ref's, restated here with token type ids (``BertEmbeddings.forward`` adds
``token_type_embeddings[token_type_ids]``; bge_ref.forward_np fixes them at 0, as every embedding model runs).  The head is
``BertPooler`` (dense + tanh on the [CLS] row of the last hidden state) then the classifier Linear: ``num_labels`` raw
logits per item (HF modeling_bert.py, BertPooler and BertForSequenceClassification.forward; dropout is the identity at
inference).  TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

import kernel_refs as KR
from oracle import bge_ref as R

HEAD_STYLES = ("hf", "trained")
CLS_B_PAD = 128  # b200rt.weights.classifier_blob_layout pads the classifier bias to 128 floats


# ------------------------------------------------------------------------------------------------ weights

def _replay_encoder_draws(rng, g, style):
    """Advance `rng` past exactly the draws R.make_weights(g, seed, style) makes (same generator, same order), so that the head
    is drawn after them and the encoder's tensors stay bit-identical to make_weights'."""
    lay = R.blob_layout(g)
    for name, shape in lay:
        if name.endswith(".w") or name.startswith("emb.") and not name.startswith("emb.ln"):
            rng.standard_normal(shape, dtype=np.float32)
    if style == "trained":
        for name, shape in lay:
            if name.endswith(".g") or name.endswith(".b"):
                rng.standard_normal(shape, dtype=np.float32)
    elif style != "hf":
        raise ValueError(f"classifier weights come in styles {HEAD_STYLES}, not {style!r}")


# `trained` head: the pooler's pre-activations at sigma ~1.5, so the tanh saturates on part of its range, and logits spread
# over about +-10 across inputs, as a trained ms-marco cross-encoder's are.  The LayerNorm'd [CLS] row has about unit scale
# per channel, so a pooler weight of sigma 1.5 / sqrt(H) gives pre-activations of sigma ~1.5.  A seeded encoder's [CLS] rows
# of different inputs differ little (the pooled vectors vary by ~0.06 per channel around a common mean), so a random
# classifier would give every input nearly the same logit.  The classifier is therefore fitted to a fixed seeded calibration
# batch: random rows mapped through the inputs' covariance (weight on the directions in which inputs differ), scaled to
# logit sigma TRAINED_LOGIT_SIGMA, and the bias set to centre the logits near 0 -- a deterministic function of the seed.
TRAINED_PRE_SIGMA = 1.5
TRAINED_LOGIT_SIGMA = 4.0
CALIB_ITEMS, CALIB_S = 32, 64


def make_classifier_weights(g: R.BertGeometry, seed: int = 0, style: str = "hf", num_labels: int = 1) -> dict:
    """R.make_weights(g, seed, style) plus the head, drawn from the same generator after make_weights' draws:
    pool.w [H, H], pool.b [H], cls.w [L, H], cls.b [L].  `hf`: sigma 0.02 matrices, zero biases -- bit-identical to
    b200rt.weights.random_classifier_blob.  `trained`: see TRAINED_PRE_SIGMA / TRAINED_LOGIT_SIGMA."""
    flat = R.make_weights(g, seed, style)
    rng = np.random.default_rng(seed)
    _replay_encoder_draws(rng, g, style)
    h, L = g.hidden, num_labels
    pw = rng.standard_normal((h, h), dtype=np.float32)
    cw = rng.standard_normal((L, h), dtype=np.float32)
    if style == "hf":
        flat.update({"pool.w": pw * np.float32(0.02), "pool.b": np.zeros(h, np.float32), "cls.w": cw * np.float32(0.02),
                     "cls.b": np.zeros(L, np.float32)})
        return flat
    pb = rng.standard_normal(h, dtype=np.float32)
    cb = rng.standard_normal(L, dtype=np.float32)
    flat["pool.w"] = (pw * np.float32(TRAINED_PRE_SIGMA / math.sqrt(h))).astype(np.float32)
    flat["pool.b"] = (pb * np.float32(0.1)).astype(np.float32)
    crng = np.random.default_rng(seed + 7919)
    lens = crng.integers(8, CALIB_S + 1, size=CALIB_ITEMS)
    segs = [int(crng.integers(2, n)) for n in lens]
    ids, lens, segs = synth_pairs(lens, segs, CALIB_S, seed + 7919, g.vocab)
    hp = pooled_np(flat, ids, lens, segs, g)
    mu = hp.mean(0)
    hc = hp - mu
    w = cw.astype(np.float64) @ (hc.T @ hc) / CALIB_ITEMS
    w *= TRAINED_LOGIT_SIGMA / np.std(hc @ w.T, axis=0)[:, None]
    flat["cls.w"] = w.astype(np.float32)
    flat["cls.b"] = (-(w @ mu) + 0.5 * cb).astype(np.float32)
    return flat


def pack_classifier_blob(flat: dict, g: R.BertGeometry) -> np.ndarray:
    """The fp32 blob of b200rt.weights.classifier_blob_layout: bge_ref's blob, then pool.w | pool.b | cls.w | cls.b padded."""
    L = flat["cls.w"].shape[0]
    cb = np.zeros(CLS_B_PAD, np.float32)
    cb[:L] = flat["cls.b"]
    return np.concatenate([R.pack_blob({k: v for k, v in flat.items() if not k.startswith(("pool.", "cls."))}, g),
                           flat["pool.w"].reshape(-1), flat["pool.b"], flat["cls.w"].reshape(-1), cb]).astype(np.float32)


def geometry_dict(g: R.BertGeometry, num_labels: int) -> dict:
    return dict(R.geometry_dict(g), num_labels=num_labels)


# ------------------------------------------------------------------------------------------------ inputs

def token_types(segs, S):
    """[B, S] token type ids: 1 from segs[i] on, 0 before."""
    return (np.arange(S)[None, :] >= np.asarray(segs)[:, None]).astype(np.int64)


def synth_pairs(lens, segs, S, seed, vocab=30522):
    """ids [len(lens), S] of [CLS] a [SEP] b [SEP] items: [SEP] at segs[i] - 1 and lens[i] - 1 (segs[i] == lens[i]: a single
    sequence), interior ids uniform in [1000, vocab), [PAD] after the length."""
    rng = np.random.default_rng(seed)
    ids = np.zeros((len(lens), S), np.int32)
    for i, (n, s) in enumerate(zip(lens, segs)):
        assert 0 <= s <= n <= S
        ids[i, :n] = rng.integers(1000, vocab, size=n)
        ids[i, 0] = 101
        ids[i, n - 1] = 102
        if 1 <= s < n:
            ids[i, s - 1] = 102
    return ids, np.asarray(lens, np.int32), np.asarray(segs, np.int32)


# ------------------------------------------------------------------------------------------------ forward (numpy)

def hidden_np(flat, ids, lens, segs, g: R.BertGeometry, dtype=np.float64):
    """Last hidden state [B, S, H] of BertModel.forward with token_type_ids from segs (None: all 0) -- bge_ref.forward_np's
    encoder with the type row chosen per token."""
    ids = np.asarray(ids)
    B, S = ids.shape
    lens = np.full(B, S, np.int32) if lens is None else np.asarray(lens)
    tt = np.zeros((B, S), np.int64) if segs is None else token_types(segs, S)
    W = {k: v.astype(dtype) for k, v in flat.items() if not k.startswith("emb.word")}
    h, nh, dh = g.hidden, g.heads, g.head_dim
    x = flat["emb.word"][ids].astype(dtype) + W["emb.type"][tt] + W["emb.pos"][:S][None]
    x = R._layer_norm(x, W["emb.ln.g"], W["emb.ln.b"], g.eps)
    keymask = np.arange(S)[None, :] >= lens[:, None]
    scale = 1.0 / math.sqrt(dh)
    for l in range(g.layers):
        p = f"l{l}."
        qkv = x @ W[p + "qkv.w"].T + W[p + "qkv.b"]
        q, k, v = (qkv[..., j * h:(j + 1) * h].reshape(B, S, nh, dh).transpose(0, 2, 1, 3) for j in range(3))
        s = (q @ k.transpose(0, 1, 3, 2)) * scale
        s = np.where(keymask[:, None, None, :], -np.inf, s)
        e = np.exp(s - s.max(-1, keepdims=True))
        ctx = ((e / e.sum(-1, keepdims=True)) @ v).transpose(0, 2, 1, 3).reshape(B, S, h)
        x = R._layer_norm(ctx @ W[p + "ao.w"].T + W[p + "ao.b"] + x, W[p + "ln1.g"], W[p + "ln1.b"], g.eps)
        y = R._gelu(x @ W[p + "ff1.w"].T + W[p + "ff1.b"])
        x = R._layer_norm(y @ W[p + "ff2.w"].T + W[p + "ff2.b"] + x, W[p + "ln2.g"], W[p + "ln2.b"], g.eps)
    return x


def pooled_np(flat, ids, lens, segs, g, dtype=np.float64):
    """BertPooler: tanh(W_p x_CLS + b_p), [B, H]."""
    x = hidden_np(flat, ids, lens, segs, g, dtype)[:, 0]
    return np.tanh(x @ flat["pool.w"].astype(dtype).T + flat["pool.b"].astype(dtype))


def classify_np(flat, ids, lens, segs, g, dtype=np.float64):
    """[B, L] raw logits: classifier(BertPooler(last hidden state)), in dtype (fp64 by default)."""
    hp = pooled_np(flat, ids, lens, segs, g, dtype)
    return hp @ flat["cls.w"].astype(dtype).T + flat["cls.b"].astype(dtype)


def pooler_preactivations(flat, ids, lens, segs, g):
    x = hidden_np(flat, ids, lens, segs, g)[:, 0]
    return x @ flat["pool.w"].astype(np.float64).T + flat["pool.b"].astype(np.float64)


# ------------------------------------------------------------------------------------------------ forward (HF torch)

def build_hf_classifier(flat: dict, g: R.BertGeometry):
    """``transformers.BertForSequenceClassification`` built from its config (no download) and loaded with `flat`."""
    import torch
    from transformers import BertConfig, BertForSequenceClassification

    L = flat["cls.w"].shape[0]
    cfg = BertConfig(vocab_size=g.vocab, hidden_size=g.hidden, num_hidden_layers=g.layers, num_attention_heads=g.heads,
                     intermediate_size=g.inter, max_position_embeddings=g.max_pos, type_vocab_size=g.type_vocab,
                     layer_norm_eps=g.eps, hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                     num_labels=L)
    with torch.device("meta"):
        model = BertForSequenceClassification(cfg)
    model = model.to_empty(device="cpu")
    enc = {k: v for k, v in flat.items() if not k.startswith(("pool.", "cls."))}
    sd = {"bert." + k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in R.flat_to_hf_state(enc, g).items()}
    sd.update({"bert.pooler.dense.weight": torch.from_numpy(flat["pool.w"]), "bert.pooler.dense.bias": torch.from_numpy(flat["pool.b"]),
               "classifier.weight": torch.from_numpy(flat["cls.w"]), "classifier.bias": torch.from_numpy(flat["cls.b"])})
    missing, unexpected = model.load_state_dict(sd, strict=False)
    missing = [m for m in missing if "position_ids" not in m and "token_type_ids" not in m]
    assert not missing and not unexpected, (missing, unexpected)
    with torch.no_grad():
        emb = model.bert.embeddings
        if hasattr(emb, "position_ids"):
            emb.position_ids = torch.arange(g.max_pos).unsqueeze(0)
        if hasattr(emb, "token_type_ids"):
            emb.token_type_ids = torch.zeros((1, g.max_pos), dtype=torch.long)
    return model.eval()


def classify_hf(model, ids, lens, segs) -> np.ndarray:
    """[B, L] fp32 logits of HF BertForSequenceClassification (CPU)."""
    import torch

    ids_t = torch.from_numpy(np.ascontiguousarray(ids)).long()
    B, S = ids_t.shape
    mask = (torch.arange(S)[None, :] < torch.from_numpy(np.asarray(lens))[:, None]).long()
    tt = torch.from_numpy(token_types(segs, S))
    with torch.no_grad():
        return model(input_ids=ids_t, attention_mask=mask, token_type_ids=tt).logits.numpy().astype(np.float32)


# ------------------------------------------------------------------------------------------------ kernel references

def embed_segs_exact(ids, segs, word, pos, type2, S):
    """embed_kernel<W, SEGS>, bit for bit: x = (word[id] + type2[t % S >= segs[t // S]]) + pos[t % S] in fp32, segs clamped to
    [0, S]; hi = fp16_rn(x), lo = fp16_rn(x - hi).  Returns (hi, lo, x)."""
    ids = np.asarray(ids).reshape(-1)
    t = np.arange(ids.size)
    sg = np.clip(np.asarray(segs, np.int64), 0, S)[t // S]
    row = (t % S >= sg).astype(np.int64)
    x = (np.asarray(word, np.float32)[ids] + np.asarray(type2, np.float32)[row]) + np.asarray(pos, np.float32)[t % S]
    hi, lo = KR.split_hilo(x)
    return hi, lo, x


def check_embed_segs(what, hi, lo, stats, ids, segs, word, pos, type2, S, rows=None):
    """hi and lo bit for bit over every row; the partials over `rows` (stats then holds those rows), by default all."""
    hi_r, lo_r, x = embed_segs_exact(ids, segs, word, pos, type2, S)
    KR.check_bits(f"{what} hi", hi, hi_r)
    KR.check_bits(f"{what} lo", lo, lo_r)
    if rows is not None:
        x = x[rows]
    return KR.check_partials(f"{what} partials", np.asarray(stats), x.astype(np.float64))


def _dot_ulps(W):
    """fp32 roundings of one head dot product: W / 32 fma per lane, 5 butterfly levels, the bias add, and margin."""
    return W / 32 + 8.0


def cls_head_ref(hi, lo, gamma, beta, pool_w, pool_b, cls_w, cls_b, S, eps):
    """(logits, tol) of cls_head_kernel on the CLS rows of hi + lo, fp64.  The LayerNorm's bound is carried through |W_p|, the
    tanh's slope (1 - h^2) and |W_c|; each dot product adds its own fp32 roundings and tanhf up to 2 ulp."""
    x = KR.hilo64(hi, lo)[::S]
    z, z_tol, _ = KR.layernorm_ref(x, gamma, beta, eps)
    wp = np.asarray(pool_w, np.float32).astype(np.float64)
    bp = np.asarray(pool_b, np.float32).astype(np.float64)
    wc = np.asarray(cls_w, np.float32).astype(np.float64)
    bc = np.asarray(cls_b, np.float32).astype(np.float64)[: wc.shape[0]]
    W = wp.shape[0]
    pre = z @ wp.T + bp
    pre_tol = z_tol @ np.abs(wp).T + _dot_ulps(W) * KR.U32 * (np.abs(z) @ np.abs(wp).T + np.abs(bp))
    h = np.tanh(pre)
    h_tol = (1.0 - h * h) * pre_tol + 3.0 * KR.U32 * np.abs(h) + 1e-30
    y = h @ wc.T + bc
    y_tol = h_tol @ np.abs(wc).T + _dot_ulps(W) * KR.U32 * (np.abs(h) @ np.abs(wc).T + np.abs(bc))
    return y, y_tol


def check_cls_head(what, out, hi, lo, gamma, beta, pool_w, pool_b, cls_w, cls_b, S, eps):
    ref, tol = cls_head_ref(hi, lo, gamma, beta, pool_w, pool_b, cls_w, cls_b, S, eps)
    return KR.check(what, out, ref, tol)


# ------------------------------------------------------------------------------------------------ emulations and mutants

EMBED_MUTANTS = ("type_ignored", "seg_off_by_one")
HEAD_MUTANTS = ("no_ln", "row1", "no_tanh", "wc_transposed", "no_pool_bias")


def emulate_embed_segs(ids, segs, word, pos, type2, S, mutant=None):
    """(hi, lo, stats) as the kernel rounds them; mutants: the type row ignored (row 0 throughout), or the second segment
    starting one token late."""
    segs = np.asarray(segs, np.int64)
    if mutant == "type_ignored":
        segs = np.full_like(segs, S)
    elif mutant == "seg_off_by_one":
        segs = segs + 1
    elif mutant is not None:
        raise ValueError(mutant)
    hi, lo, x = embed_segs_exact(ids, segs, word, pos, type2, S)
    from kernel_emul import partials32

    return hi, lo, partials32(x)


def emulate_cls_head(hi, lo, gamma, beta, pool_w, pool_b, cls_w, cls_b, S, eps, mutant=None):
    """The head in fp32, rounding as the kernel rounds (fp32 LayerNorm, fp32 dot products, tanhf); mutants: no LayerNorm, row 1
    instead of the CLS row, no tanh, W_c read transposed, no pooler bias."""
    x = (np.asarray(hi, np.float16).astype(np.float32) + np.asarray(lo, np.float16).astype(np.float32))
    x = x[1::S] if mutant == "row1" else x[::S]
    g32, b32 = np.asarray(gamma, np.float32), np.asarray(beta, np.float32)
    if mutant == "no_ln":
        z = x
    else:
        mu = x.mean(-1, keepdims=True, dtype=np.float32)
        d = x - mu
        rstd = np.float32(1.0) / np.sqrt((d * d).mean(-1, keepdims=True, dtype=np.float32) + np.float32(eps))
        z = (d * rstd) * g32 + b32
    wp = np.asarray(pool_w, np.float32)
    bp = np.zeros_like(pool_b, dtype=np.float32) if mutant == "no_pool_bias" else np.asarray(pool_b, np.float32)
    pre = (z @ wp.T).astype(np.float32) + bp
    h = pre if mutant == "no_tanh" else np.tanh(pre).astype(np.float32)
    wc = np.asarray(cls_w, np.float32)
    L, W = wc.shape
    if mutant == "wc_transposed":
        wc = wc.reshape(-1).reshape(W, L).T
    return ((h @ wc.T).astype(np.float32) + np.asarray(cls_b, np.float32)[:L]).astype(np.float32)


# ------------------------------------------------------------------------------------------------ fp16-operand emulation

def classify_fp16_operands(flat, ids, lens, segs, g):
    """The forward with the rounding the GPU path cannot avoid, everything else fp64: every GEMM operand (activations and
    weights) and the attention's Q, K, V and probabilities rounded to fp16, the residual stream kept to hi + lo.  Its distance
    from classify_np is the floor of any GPU-vs-oracle comparison."""
    f16 = lambda a: np.asarray(a, np.float64).astype(np.float16).astype(np.float64)  # noqa: E731
    hl = lambda a: f16(a) + f16(np.asarray(a, np.float64) - f16(a))  # noqa: E731
    ids = np.asarray(ids)
    B, S = ids.shape
    lens = np.asarray(lens)
    tt = token_types(segs, S)
    W = {k: np.asarray(v, np.float64) for k, v in flat.items() if not k.startswith("emb.word")}
    h, nh, dh = g.hidden, g.heads, g.head_dim
    y = hl(flat["emb.word"][ids].astype(np.float64) + W["emb.type"][tt] + W["emb.pos"][:S][None])
    ln = lambda v, a, b: R._layer_norm(v, W[a], W[b], g.eps)  # noqa: E731
    x = ln(y, "emb.ln.g", "emb.ln.b")
    keymask = np.arange(S)[None, :] >= lens[:, None]
    for l in range(g.layers):
        p = f"l{l}."
        qkv = f16(f16(x) @ f16(W[p + "qkv.w"]).T + W[p + "qkv.b"])
        q, k, v = (qkv[..., j * h:(j + 1) * h].reshape(B, S, nh, dh).transpose(0, 2, 1, 3) for j in range(3))
        s = (q @ k.transpose(0, 1, 3, 2)) / math.sqrt(dh)
        s = np.where(keymask[:, None, None, :], -np.inf, s)
        e = np.exp(s - s.max(-1, keepdims=True))
        pr = e / e.sum(-1, keepdims=True)
        ctx = f16((f16(pr) @ v).transpose(0, 2, 1, 3).reshape(B, S, h))
        x = ln(hl(ctx @ f16(W[p + "ao.w"]).T + W[p + "ao.b"] + x), p + "ln1.g", p + "ln1.b")
        a = f16(R._gelu(f16(x) @ f16(W[p + "ff1.w"]).T + W[p + "ff1.b"]))
        x = ln(hl(a @ f16(W[p + "ff2.w"]).T + W[p + "ff2.b"] + x), p + "ln2.g", p + "ln2.b")
    hp = np.tanh(x[:, 0] @ W["pool.w"].T + W["pool.b"])
    return hp @ W["cls.w"].T + W["cls.b"]
