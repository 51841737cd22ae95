"""fp64 oracle of SPLADE sparse encoders (HF ``BertForMaskedLM`` + sentence-transformers' ``SpladePooling(max, relu)``, as TEI
runs ``--pooling splade``), the kernel references of the SPLADE head's launches, numpy emulations of them with the mutants
their checks must reject, and the fp16-operand emulation that sets the parity floor.

For item i with lens[i] valid tokens and h_t the final hidden state of token t:
    u_t = gelu_erf(W_t h_t + b_t);  z_t = LN_t(u_t);  logit_t = W_dec z_t + b_dec
    out[i] = max_{t < lens[i]} log1p(relu(logit_t)) = log1p(max(0, max_t logit_t))          [vocab], unnormalised
(HF modeling_bert.py BertPredictionHeadTransform / BertLMPredictionHead; the decoder is tied to the word embeddings).
The encoder is rerank_refs.hidden_np's (oracle/bge_ref's with token types; every token here is type 0).
TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

import kernel_refs as KR
import rerank_refs as RR
from oracle import bge_ref as R

STYLES = ("hf", "splade")
U32 = 2.0 ** -24


def vpad(vocab: int) -> int:
    """The decoder GEMM's width: the vocabulary tiled to 256 columns."""
    return (vocab + 255) // 256 * 256


# ------------------------------------------------------------------------------------------------ weights

# `splade` head: a trained SPLADE document vector keeps roughly 50-400 non-zero words for a 64-256-token input, with values
# up to ~2-3.  The transform LayerNorm's gain is raised so the logits spread with sigma ~SPLADE_LOGIT_SIGMA, and b_dec is a
# negative constant, fitted on a fixed seeded calibration batch so that its median item keeps SPLADE_NNZ words.
SPLADE_LOGIT_SIGMA = 2.0
SPLADE_NNZ = 150
CALIB_ITEMS, CALIB_S = 6, 128


def make_splade_weights(g: R.BertGeometry, seed: int = 0, style: str = "hf") -> dict:
    """R.make_weights(g, seed, "hf" or "trained" for style `splade`) plus the masked-LM head, drawn from the same generator
    after make_weights' draws: mlm.t.w [H, H], mlm.t.b [H], mlm.ln.g / mlm.ln.b [H], mlm.dec.w [V, H] (tied: the word embeddings),
    mlm.dec.b [V].  `hf`: HF init (sigma 0.02, zero biases, unit LayerNorm): about half the vocabulary ends up non-zero.
    `splade`: see SPLADE_LOGIT_SIGMA / SPLADE_NNZ."""
    if style not in STYLES:
        raise ValueError(f"SPLADE weights come in styles {STYLES}, not {style!r}")
    enc_style = "hf" if style == "hf" else "trained"
    flat = R.make_weights(g, seed, enc_style)
    rng = np.random.default_rng(seed)
    RR._replay_encoder_draws(rng, g, enc_style)
    h = g.hidden
    tw = rng.standard_normal((h, h), dtype=np.float32)
    flat["mlm.t.w"] = tw * np.float32(0.02)
    flat["mlm.t.b"] = np.zeros(h, np.float32)
    flat["mlm.ln.g"] = np.ones(h, np.float32)
    flat["mlm.ln.b"] = np.zeros(h, np.float32)
    flat["mlm.dec.w"] = flat["emb.word"]
    flat["mlm.dec.b"] = np.zeros(g.vocab, np.float32)
    if style == "hf":
        return flat
    tb = rng.standard_normal(h, dtype=np.float32)
    lg = rng.standard_normal(h, dtype=np.float32)
    lb = rng.standard_normal(h, dtype=np.float32)
    flat["mlm.t.w"] = (tw * np.float32(1.0 / math.sqrt(h))).astype(np.float32)
    flat["mlm.t.b"] = (0.1 * tb).astype(np.float32)
    dec_sigma = float(np.std(flat["emb.word"])) * math.sqrt(h)  # a unit LayerNorm'd z gives logits of this sigma
    flat["mlm.ln.g"] = (SPLADE_LOGIT_SIGMA / dec_sigma * (1.0 + 0.1 * lg)).astype(np.float32)
    flat["mlm.ln.b"] = (0.05 * lb).astype(np.float32)
    ids, lens = calib_batch(g, seed)
    mx = item_max_logits(flat, ids, lens, g)  # [items, V], b_dec = 0
    kth = np.sort(mx, axis=1)[:, g.vocab - SPLADE_NNZ]
    flat["mlm.dec.b"] = np.full(g.vocab, -float(np.median(kth)), np.float32)
    return flat


def calib_batch(g: R.BertGeometry, seed: int):
    return R.synth_ragged(CALIB_ITEMS, CALIB_S, seed=seed + 7919, min_len=64, vocab=g.vocab)


def pack_splade_blob(flat: dict, g: R.BertGeometry) -> np.ndarray:
    """The fp32 blob of b200rt.weights.splade_blob_layout: bge_ref's blob, then the head, the decoder bias padded to 128."""
    db = np.zeros((g.vocab + 127) // 128 * 128, np.float32)
    db[: g.vocab] = flat["mlm.dec.b"]
    enc = {k: v for k, v in flat.items() if not k.startswith("mlm.")}
    return np.concatenate([R.pack_blob(enc, g), flat["mlm.t.w"].reshape(-1), flat["mlm.t.b"], flat["mlm.ln.g"], flat["mlm.ln.b"],
                           flat["mlm.dec.w"].reshape(-1), db]).astype(np.float32)


# ------------------------------------------------------------------------------------------------ forward (numpy)

def _head_z(flat, h, eps, dtype=np.float64):
    """LN_t(gelu(W_t h + b_t)) of hidden rows h [n, H]."""
    W = lambda k: flat[k].astype(dtype)  # noqa: E731
    u = R._gelu(h @ W("mlm.t.w").T + W("mlm.t.b"))
    return R._layer_norm(u, W("mlm.ln.g"), W("mlm.ln.b"), eps)


def item_max_logits(flat, ids, lens, g, dtype=np.float64):
    """[B, V]: max over each item's valid tokens of its MLM logits (before relu)."""
    hid = RR.hidden_np(flat, ids, lens, None, g, dtype)
    dec = flat["mlm.dec.w"].astype(dtype)
    b = flat["mlm.dec.b"].astype(dtype)
    out = np.empty((len(lens), g.vocab), dtype)
    for i, n in enumerate(np.asarray(lens)):
        z = _head_z(flat, hid[i, :n], g.eps, dtype)
        out[i] = (z @ dec.T + b).max(0)
    return out


def splade_np(flat, ids, lens, g, dtype=np.float64):
    """[B, V] SPLADE vectors, fp64 by default."""
    return np.log1p(np.maximum(item_max_logits(flat, ids, lens, g, dtype), 0.0))


def splade_fp16_operands(flat, ids, lens, g):
    """The oracle with the head's GEMM operands rounded to fp16 as the GPU path feeds them (the last hidden state, u, the
    folded W_t and W_dec''), everything else fp64: the precision floor of the head alone, for the parity bar."""
    hid = RR.hidden_np(flat, ids, lens, None, g)
    f16 = lambda x: np.asarray(x).astype(np.float16).astype(np.float64)  # noqa: E731
    W = lambda k: flat[k].astype(np.float64)  # noqa: E731
    wt, wd = W("mlm.t.w"), W("mlm.dec.w")
    out = np.empty((len(lens), g.vocab))
    for i, n in enumerate(np.asarray(lens)):
        u = R._gelu(f16(hid[i, :n]) @ f16(wt).T + W("mlm.t.b"))
        u = f16(u)
        mu = u.mean(-1, keepdims=True)
        rstd = 1.0 / np.sqrt(((u - mu) ** 2).mean(-1, keepdims=True) + g.eps)
        wg = wd * W("mlm.ln.g")
        wg = f16(wg - wg.mean(1, keepdims=True))
        logit = rstd * (u @ wg.T) + (wd @ W("mlm.ln.b") + W("mlm.dec.b"))
        out[i] = np.log1p(np.maximum(logit.max(0), 0.0))
    return out


# ------------------------------------------------------------------------------------------------ forward (HF torch)

def build_hf_masked_lm(flat: dict, g: R.BertGeometry):
    """``transformers.BertForMaskedLM`` built from its config (no download), loaded with `flat`, its decoder tied to the word
    embeddings as HF ties it (so `flat`'s mlm.dec.w must be emb.word)."""
    import torch
    from transformers import BertConfig, BertForMaskedLM

    assert np.array_equal(flat["mlm.dec.w"], flat["emb.word"]), "HF ties the decoder to the word embeddings"
    cfg = BertConfig(vocab_size=g.vocab, hidden_size=g.hidden, num_hidden_layers=g.layers, num_attention_heads=g.heads,
                     intermediate_size=g.inter, max_position_embeddings=g.max_pos, type_vocab_size=g.type_vocab,
                     layer_norm_eps=g.eps, hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                     tie_word_embeddings=True)
    model = BertForMaskedLM(cfg)
    enc = {k: v for k, v in flat.items() if not k.startswith("mlm.")}
    sd = {"bert." + k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in R.flat_to_hf_state(enc, g).items()}
    t = "cls.predictions.transform."
    sd.update({t + "dense.weight": torch.from_numpy(flat["mlm.t.w"]), t + "dense.bias": torch.from_numpy(flat["mlm.t.b"]),
               t + "LayerNorm.weight": torch.from_numpy(flat["mlm.ln.g"]), t + "LayerNorm.bias": torch.from_numpy(flat["mlm.ln.b"]),
               "cls.predictions.bias": torch.from_numpy(flat["mlm.dec.b"])})
    missing, unexpected = model.load_state_dict(sd, strict=False)
    missing = [m for m in missing if "position_ids" not in m and "token_type_ids" not in m and "decoder" not in m]
    assert not missing and not unexpected, (missing, unexpected)
    model.tie_weights()
    assert model.cls.predictions.decoder.weight.data_ptr() == model.bert.embeddings.word_embeddings.weight.data_ptr()
    return model.eval()


def splade_hf(model, ids, lens) -> np.ndarray:
    """[B, V] fp32 SPLADE vectors of HF BertForMaskedLM (CPU): SpladePooling(max, relu) = max over the attended tokens of
    log1p(relu(logits))."""
    import torch

    ids_t = torch.from_numpy(np.ascontiguousarray(ids)).long()
    B, S = ids_t.shape
    mask = (torch.arange(S)[None, :] < torch.from_numpy(np.asarray(lens))[:, None]).long()
    out = []
    with torch.no_grad():
        for i in range(B):
            logits = model(input_ids=ids_t[i:i + 1], attention_mask=mask[i:i + 1], token_type_ids=torch.zeros_like(ids_t[i:i + 1])).logits
            v = torch.log1p(torch.relu(logits[0])) * mask[i][:, None]
            out.append(v.max(0).values.numpy())
    return np.stack(out).astype(np.float32)


# ------------------------------------------------------------------------------------------------ kernel references

def gemm_splade_ref(a16, w16, c, stats, lens, S, N, eps):
    """What b200rt_debug_gemm_splade returns, as fp32 values (the maxima's bits read as floats), and its tolerance, fp64, both
    [B, N]: max(0, max over item i's valid rows of rstd_r (a_r . w_n) + c_n) for n < vocab, 0 past it.  The bound of a max
    is the largest bound among the rows it ranges over."""
    lens = np.asarray(lens)
    B = len(lens)
    vocab = w16.shape[0]
    v, _, v_tol = KR.gemm_ref(0, a16, w16, np.asarray(c, np.float32)[:vocab], ln_stats=stats, eps=eps)
    ref = np.zeros((B, N))
    tol = np.zeros((B, N))
    for i in range(B):
        n = int(min(max(lens[i], 0), S))
        if n == 0:
            continue
        rows = slice(i * S, i * S + n)
        ref[i, :vocab] = np.maximum(v[rows].max(0), 0.0)
        tol[i, :vocab] = v_tol[rows].max(0)
    return ref, tol


def check_gemm_splade(what, vmax_bits, a16, w16, c, stats, lens, S, eps):
    """The maxima against gemm_splade_ref: within tolerance for n < vocab, and every word past vocab exactly 0 (never written)."""
    vmax_bits = np.asarray(vmax_bits, np.uint32)
    B, N = vmax_bits.shape
    vocab = w16.shape[0]
    assert not vmax_bits[:, vocab:].any(), f"{what}: a column >= vocab was written"
    got = vmax_bits.view(np.float32).astype(np.float64)
    ref, tol = gemm_splade_ref(a16, w16, c, stats, lens, S, N, eps)
    return KR.check(what, got[:, :vocab], ref[:, :vocab], tol[:, :vocab])


def emulate_gemm_splade(a16, w16, c, stats, lens, S, N, eps, mutant=None):
    """uint32 [B, N] maxima as the kernel forms them (fp32 epilogue on fp64 dot products, integer max of the bits), or a mutant:
    pad_row   -- one padded row included (len off by one);
    neighbour -- the second 64-row half of each item's rows credited to the next item;
    no_relu   -- relu dropped before the integer max (a negative's bits exceed every positive's);
    no_stats  -- u's statistics not applied (rstd = 1);
    shift8    -- columns shifted by 8;
    past_vocab -- columns >= vocab written."""
    from kernel_emul import row_stats32

    lens = np.clip(np.asarray(lens), 0, S)
    B = len(lens)
    vocab = w16.shape[0]
    acc = (np.asarray(a16, np.float16).astype(np.float64) @ np.asarray(w16, np.float16).astype(np.float64).T).astype(np.float32)
    _, rstd = row_stats32(np.asarray(stats, np.float32), eps)
    if mutant == "no_stats":
        rstd = np.ones_like(rstd)
    cc = np.asarray(c, np.float32)[:vocab]
    v = (rstd[:, None].astype(np.float32) * acc + cc).astype(np.float32)
    if mutant == "past_vocab":
        v = np.concatenate([v, np.full((v.shape[0], N - vocab), 1.0, np.float32)], 1)
    out = np.zeros((B, N), np.uint32)
    for i in range(B):
        n = int(lens[i]) + (1 if mutant == "pad_row" else 0)
        n = min(n, S)
        if n == 0:
            continue
        rows = v[i * S: i * S + n]
        if mutant == "no_relu":
            m = rows.view(np.uint32).max(0)
        else:
            m = np.maximum(rows.max(0), np.float32(0)).view(np.uint32)
        out[i, : m.size] = np.maximum(out[i, : m.size], m)
        if mutant == "neighbour" and i + 1 < B and n > 64:
            out[i + 1, : m.size] = np.maximum(out[i + 1, : m.size], np.maximum(rows[64:].max(0), 0).astype(np.float32).view(np.uint32))
    if mutant == "shift8":
        out = np.roll(out, 8, axis=1)
        out[:, vocab:] = 0
    return out


def splade_finalize_ref(vmax_bits, vocab):
    """(log1p of the maxima read as fp32, tolerance 2 fp32 ulps of the result): log1pf is within 1 ulp."""
    x = np.asarray(vmax_bits, np.uint32)[:, :vocab].view(np.float32).astype(np.float64)
    r = np.log1p(x)
    return r, 2.0 * U32 * np.abs(r) + 1e-45


def check_splade_finalize(what, out, vmax_bits, vocab):
    r, tol = splade_finalize_ref(vmax_bits, vocab)
    return KR.check(what, out, r, tol)


def emulate_splade_finalize(vmax_bits, vocab, mutant=None):
    """float32 [n, vocab]: np.log1p in fp32, or (mutant `logf`) log(1 + x) with the sum rounded to fp32 first, as __logf(1 + x)
    computes it -- every value below 2^-24 becomes 0 and small ones lose their relative precision."""
    x = np.asarray(vmax_bits, np.uint32)[:, :vocab].view(np.float32)
    if mutant == "logf":
        return np.log((np.float32(1) + x).astype(np.float32)).astype(np.float32)
    return np.log1p(x.astype(np.float64)).astype(np.float32)


def finalize_probe(n_items=3, vpad=512, vocab=500, seed=0):
    """uint32 maxima whose values cover the range log1pf must keep: 0, subnormals, 1e-30 .. 1e-6 (where 1 + x rounds to 1),
    and ordinary values up to 20."""
    rng = np.random.default_rng(seed)
    x = np.zeros((n_items, vpad), np.float32)
    x[:, :vocab] = np.exp(rng.uniform(np.log(1e-30), np.log(20.0), size=(n_items, vocab))).astype(np.float32)
    x[:, :vocab][rng.random((n_items, vocab)) < 0.3] = 0.0
    x[0, :4] = np.array([1e-45, 1e-40, 3e-8, 5e-8], np.float32)
    return x.view(np.uint32)
