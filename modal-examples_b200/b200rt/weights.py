"""Product-side weight handling for ``b200rt_model_load``: the flat fp32 blob layout, the mapping from a Hugging Face
``BertModel`` checkpoint (state dict or ``model.safetensors``) to it, and seeded random weights of a geometry.

This is what stands in for the reference's ``download_model`` (``06_gpu_and_ml/embeddings/text_embeddings_inference.py:54-56``,
``snapshot_download(MODEL_ID)`` into the HF hub cache) + TEI's own weight loading: a user holding the real
``BAAI/bge-base-en-v1.5`` files calls :func:`load_safetensors` (or :func:`load_hf_dir` on the snapshot directory) and
hands the blob to :class:`b200rt.EmbedModel`.

Blob order (all fp32, HF shapes, ``y = x W^T + b`` with W ``[out, in]`` row-major; Q, K, V stacked into one ``[3H, H]``):
``emb.word [V,H] | emb.pos [P,H] | emb.type [T,H] | emb.ln.g | emb.ln.b`` then per layer
``qkv.w [3H,H] | qkv.b | ao.w [H,H] | ao.b | ln1.g | ln1.b | ff1.w [I,H] | ff1.b | ff2.w [H,I] | ff2.b | ln2.g | ln2.b``.
"""
from __future__ import annotations

import json
import os
import struct

import numpy as np

BGE_BASE_GEOMETRY = dict(vocab=30522, hidden=768, layers=12, heads=12, inter=3072, max_pos=512, type_vocab=2, eps=1e-12)
# BAAI/bge-small-en-v1.5: 12 heads of 32 -- the head count is not implied by the tensor shapes (384 // 64 would be 6)
BGE_SMALL_GEOMETRY = dict(vocab=30522, hidden=384, layers=12, heads=12, inter=1536, max_pos=512, type_vocab=2, eps=1e-12)
# sentence-transformers/all-MiniLM-L6-v2: bge-small's geometry with 6 layers; mean-pooled (see pooling_from_dir)
MINILM_L6_GEOMETRY = dict(vocab=30522, hidden=384, layers=6, heads=12, inter=1536, max_pos=512, type_vocab=2, eps=1e-12)
# BAAI/bge-large-en-v1.5 (BERT-large): 16 heads of 64, 24 layers; also the shape of e5-large-v2, gte-large, mxbai-embed-large-v1
BGE_LARGE_GEOMETRY = dict(vocab=30522, hidden=1024, layers=24, heads=16, inter=4096, max_pos=512, type_vocab=2, eps=1e-12)
# cross-encoder/ms-marco-MiniLM-L-6-v2 (BertForSequenceClassification): MiniLM-L6's encoder, a pooler and one relevance logit;
# -L-12-v2 is the same with 12 layers
MS_MARCO_MINILM_L6_GEOMETRY = dict(MINILM_L6_GEOMETRY, num_labels=1)

_ST_POOLING_MODULE = "sentence_transformers.models.Pooling"
_ST_POOLING_MODES = ("pooling_mode_cls_token", "pooling_mode_mean_tokens", "pooling_mode_max_tokens",
                     "pooling_mode_mean_sqrt_len_tokens", "pooling_mode_weightedmean_tokens", "pooling_mode_lasttoken")


def pooling_from_dir(path: str) -> str | None:
    """The pooling a sentence-transformers snapshot declares: ``modules.json`` names the
    ``sentence_transformers.models.Pooling`` module and its directory (``1_Pooling``), whose ``config.json`` switches the
    modes on.  Returns "cls" or "mean"; None when the directory carries no such module (a plain HF checkpoint).  Any other
    mode (max, mean_sqrt_len, weightedmean, lasttoken), or more than one at once, raises ValueError: the runtime pools the
    two supported ways only, and serving such a model with either would return a different embedding."""
    mod_path = os.path.join(path, "modules.json")
    if not os.path.exists(mod_path):
        return None
    with open(mod_path) as f:
        modules = json.load(f)
    pool = next((m for m in modules if m.get("type") == _ST_POOLING_MODULE), None)
    if pool is None:
        return None
    cfg_path = os.path.join(path, pool.get("path", ""), "config.json")
    if not os.path.exists(cfg_path):
        return None
    with open(cfg_path) as f:
        cfg = json.load(f)
    on = [k for k in _ST_POOLING_MODES if cfg.get(k)]
    if on == ["pooling_mode_cls_token"]:
        return "cls"
    if on == ["pooling_mode_mean_tokens"]:
        return "mean"
    raise ValueError(f"{cfg_path}: pooling modes {on or 'none'} enabled; the supported poolings are cls "
                     "(pooling_mode_cls_token) and mean (pooling_mode_mean_tokens), one at a time")


def blob_layout(g: dict) -> list[tuple[str, tuple[int, ...]]]:
    h, i = g["hidden"], g["inter"]
    lay = [("emb.word", (g["vocab"], h)), ("emb.pos", (g["max_pos"], h)), ("emb.type", (g["type_vocab"], h)),
           ("emb.ln.g", (h,)), ("emb.ln.b", (h,))]
    for l in range(g["layers"]):
        p = f"l{l}."
        lay += [(p + "qkv.w", (3 * h, h)), (p + "qkv.b", (3 * h,)), (p + "ao.w", (h, h)), (p + "ao.b", (h,)),
                (p + "ln1.g", (h,)), (p + "ln1.b", (h,)), (p + "ff1.w", (i, h)), (p + "ff1.b", (i,)),
                (p + "ff2.w", (h, i)), (p + "ff2.b", (h,)), (p + "ln2.g", (h,)), (p + "ln2.b", (h,))]
    return lay


def blob_numel(g: dict) -> int:
    return sum(int(np.prod(s)) for _, s in blob_layout(g))


def random_blob(g: dict = BGE_BASE_GEOMETRY, seed: int = 0) -> np.ndarray:
    """HF default init (normal sigma 0.02, zero biases, unit LayerNorm) drawn tensor by tensor, in blob order, from
    ``numpy.random.default_rng(seed)`` -- the workload weights of BASELINE.md section 3 (bit-identical to the oracle's
    ``pack_blob(make_weights(g, seed, "hf"))``, which tests/test_weights.py checks)."""
    return _random_blob(blob_layout(g), seed)


def _random_blob(layout: list, seed: int) -> np.ndarray:
    """Seeded weights of a layout, drawn tensor by tensor in blob order: unit LayerNorm gains (``.g``), zero biases and
    LayerNorm offsets (``.b``), normal sigma 0.02 matrices and embeddings (everything else)."""
    rng = np.random.default_rng(seed)
    out = np.empty(sum(int(np.prod(s)) for _, s in layout), np.float32)
    o = 0
    for name, shape in layout:
        n = int(np.prod(shape))
        if name.endswith(".g"):
            out[o:o + n] = 1.0
        elif name.endswith(".b"):
            out[o:o + n] = 0.0
        else:
            out[o:o + n] = (rng.standard_normal(shape, dtype=np.float32) * np.float32(0.02)).reshape(-1)
        o += n
    return out


def _arr(v) -> np.ndarray:
    """A numpy array or torch tensor of any float dtype as a contiguous fp32 numpy array."""
    if hasattr(v, "detach"):  # torch tensor
        v = v.detach().to("cpu").float().numpy()
    return np.ascontiguousarray(v, dtype=np.float32)


def _pack(layout: list, tensors: dict) -> np.ndarray:
    """The fp32 blob of ``layout`` from ``{layout name: tensor}``; each tensor must have its entry's shape."""
    out = np.empty(sum(int(np.prod(s)) for _, s in layout), np.float32)
    o = 0
    for name, shape in layout:
        a = _arr(tensors[name])
        if a.shape != tuple(shape):
            raise ValueError(f"checkpoint tensor has shape {a.shape}, geometry needs {tuple(shape)}")
        out[o:o + a.size] = a.reshape(-1)
        o += a.size
    return out


def _strip_prefix(sd: dict) -> dict:
    """Accept ``BertModel`` keys (``embeddings.*``), ``BertFor*`` keys (``bert.embeddings.*``) and sentence-transformers'
    ``0.auto_model.*``."""
    for pref in ("", "bert.", "0.auto_model.", "model.", "auto_model."):
        if pref + "embeddings.word_embeddings.weight" in sd:
            return {k[len(pref):]: v for k, v in sd.items() if k.startswith(pref)}
    raise KeyError("no BERT encoder weights found (looked for [bert.]embeddings.word_embeddings.weight)")


def geometry_from_state_dict(sd: dict, eps: float = 1e-12, heads: int | None = None) -> dict:
    """``heads``: ``num_attention_heads`` from the checkpoint's config.json.  Without it the head count is guessed as
    hidden // 64, which is right for bge-base; for hidden 384 that guess (6 heads of 64) is not bge-small's 12 heads of 32,
    so it raises instead."""
    sd = _strip_prefix(sd)
    vocab, hidden = sd["embeddings.word_embeddings.weight"].shape
    if heads is None and hidden == 384:
        raise ValueError("hidden 384 without num_attention_heads: bge-small has 12 heads of 32, not 384 // 64 = 6; "
                         "put the checkpoint's config.json next to its weights")
    layers = 0
    while f"encoder.layer.{layers}.attention.self.query.weight" in sd:
        layers += 1
    return dict(vocab=int(vocab), hidden=int(hidden), layers=layers, heads=int(heads or hidden // 64),
                inter=int(sd["encoder.layer.0.intermediate.dense.weight"].shape[0]),
                max_pos=int(sd["embeddings.position_embeddings.weight"].shape[0]),
                type_vocab=int(sd["embeddings.token_type_embeddings.weight"].shape[0]), eps=float(eps))


def load_hf_state_dict(sd: dict, g: dict | None = None) -> tuple[dict, np.ndarray]:
    """HF ``BertModel`` state dict (values: numpy arrays or torch tensors, any float dtype) -> (geometry, fp32 blob).
    Restates the parameter naming of HF ``modeling_bert.py`` (BertEmbeddings :72-111, BertSelfAttention :143-207,
    BertSelfOutput :287-298, BertIntermediate :330-342, BertOutput :345-356)."""
    sd = _strip_prefix(sd)
    g = dict(g) if g is not None else geometry_from_state_dict(sd)
    t = {"emb.word": sd["embeddings.word_embeddings.weight"], "emb.pos": sd["embeddings.position_embeddings.weight"],
         "emb.type": sd["embeddings.token_type_embeddings.weight"], "emb.ln.g": sd["embeddings.LayerNorm.weight"],
         "emb.ln.b": sd["embeddings.LayerNorm.bias"]}
    for l in range(g["layers"]):
        s, p = f"encoder.layer.{l}.", f"l{l}."
        t[p + "qkv.w"] = np.concatenate([_arr(sd[s + f"attention.self.{n}.weight"]) for n in ("query", "key", "value")], 0)
        t[p + "qkv.b"] = np.concatenate([_arr(sd[s + f"attention.self.{n}.bias"]) for n in ("query", "key", "value")], 0)
        t.update({p + name: sd[s + hf] for name, hf in _BERT_LAYER.items()})
    return g, _pack(blob_layout(g), t)


# a BERT layer's tensors other than Q, K, V: layout name -> HF name under encoder.layer.N.
_BERT_LAYER = {"ao.w": "attention.output.dense.weight", "ao.b": "attention.output.dense.bias",
               "ln1.g": "attention.output.LayerNorm.weight", "ln1.b": "attention.output.LayerNorm.bias",
               "ff1.w": "intermediate.dense.weight", "ff1.b": "intermediate.dense.bias",
               "ff2.w": "output.dense.weight", "ff2.b": "output.dense.bias",
               "ln2.g": "output.LayerNorm.weight", "ln2.b": "output.LayerNorm.bias"}


_ST_DTYPES = {"F32": np.float32, "F16": np.float16, "F64": np.float64, "I64": np.int64, "I32": np.int32, "U8": np.uint8}


def read_safetensors(path: str) -> dict:
    """Minimal safetensors reader (8-byte little-endian header length, JSON header, raw little-endian tensors): the
    format of the ``model.safetensors`` the reference's ``snapshot_download`` fetches.  BF16 tensors are widened to fp32."""
    with open(path, "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        header = json.loads(f.read(n))
        base = 8 + n
        out = {}
        for name, meta in header.items():
            if name == "__metadata__":
                continue
            b0, b1 = meta["data_offsets"]
            f.seek(base + b0)
            raw = f.read(b1 - b0)
            if meta["dtype"] == "BF16":
                u16 = np.frombuffer(raw, dtype="<u2").astype(np.uint32) << 16
                a = u16.view(np.float32)
            else:
                a = np.frombuffer(raw, dtype=np.dtype(_ST_DTYPES[meta["dtype"]]).newbyteorder("<"))
            out[name] = a.reshape(meta["shape"])
        return out


def write_safetensors(path: str, tensors: dict) -> None:
    """Inverse of :func:`read_safetensors` for fp32/fp16 arrays (used by the round-trip test and by tools that export
    seeded weights in the format the reference's loader expects)."""
    names = {np.dtype(np.float32): "F32", np.dtype(np.float16): "F16", np.dtype(np.int64): "I64"}
    header, blobs, off = {}, [], 0
    for name, a in tensors.items():
        a = np.ascontiguousarray(a)
        header[name] = {"dtype": names[a.dtype], "shape": list(a.shape), "data_offsets": [off, off + a.nbytes]}
        blobs.append(a.tobytes())
        off += a.nbytes
    hj = json.dumps(header, separators=(",", ":")).encode()
    hj += b" " * ((8 - len(hj) % 8) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(hj)))
        f.write(hj)
        for b in blobs:
            f.write(b)


def load_safetensors(path: str, eps: float | None = None) -> tuple[dict, np.ndarray]:
    """``model.safetensors`` of a BERT encoder -> (geometry, blob).  ``eps``/heads come from the sibling ``config.json``
    when present (``layer_norm_eps``, ``num_attention_heads``)."""
    sd = read_safetensors(path)
    cfg_path = os.path.join(os.path.dirname(os.path.abspath(path)), "config.json")
    heads = None
    if os.path.exists(cfg_path):
        cfg = json.load(open(cfg_path))
        eps = cfg.get("layer_norm_eps", eps) if eps is None else eps
        heads = cfg.get("num_attention_heads")
    g = geometry_from_state_dict(sd, eps if eps is not None else 1e-12, heads)
    return load_hf_state_dict(sd, g)


def hf_architectures(path: str) -> list:
    """``architectures`` of a snapshot directory's ``config.json`` ([] without one)."""
    p = os.path.join(path, "config.json")
    if not os.path.exists(p):
        return []
    with open(p) as f:
        return list(json.load(f).get("architectures") or [])


def load_hf_dir(path: str) -> tuple[dict, np.ndarray]:
    """A local HF snapshot directory (what ``--huggingface-hub-cache`` + ``--model-id`` resolve to): picks
    ``model.safetensors``, else ``pytorch_model.bin`` (needs torch).  A snapshot whose ``config.json`` names
    ``BertForSequenceClassification`` loads as a classifier: the geometry then carries ``num_labels`` and ``id2label``
    (the config's, else ``LABEL_i``) and the blob is :func:`classifier_blob_layout`'s."""
    cfg_path = os.path.join(path, "config.json")
    cfg = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
    st = os.path.join(path, "model.safetensors")
    pt = os.path.join(path, "pytorch_model.bin")
    if os.path.exists(st):
        sd = read_safetensors(st)
    elif os.path.exists(pt):
        import torch

        sd = torch.load(pt, map_location="cpu", weights_only=True)
    else:
        raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin under {path}")
    if CLASSIFIER_ARCHITECTURE in (cfg.get("architectures") or []):
        return load_hf_classifier(sd, cfg)
    return load_hf_state_dict(sd, geometry_from_state_dict(sd, cfg.get("layer_norm_eps", 1e-12), cfg.get("num_attention_heads")))


# ----------------------------------------------------------------------------------------------- BERT sequence classifiers
# Cross-encoders such as cross-encoder/ms-marco-MiniLM-L-6-v2 (HF BertForSequenceClassification), which TEI serves through
# /rerank and /predict.  Blob order: blob_layout(g), then pool.w [H,H] | pool.b [H] | cls.w [L,H] | cls.b [128] -- the
# classifier bias padded with zeros to 128 floats, as the engine's loader keeps every tensor a whole number of 128 floats.

CLASSIFIER_ARCHITECTURE = "BertForSequenceClassification"
CLS_B_PAD = 128


def default_id2label(num_labels: int) -> dict:
    return {i: f"LABEL_{i}" for i in range(num_labels)}


def classifier_blob_layout(g: dict) -> list[tuple[str, tuple[int, ...]]]:
    h, L = g["hidden"], g["num_labels"]
    if not 1 <= L <= 64:
        raise ValueError(f"num_labels {L} outside [1, 64]")
    return blob_layout(g) + [("pool.w", (h, h)), ("pool.b", (h,)), ("cls.w", (L, h)), ("cls.b", (CLS_B_PAD,))]


def random_classifier_blob(g: dict = MS_MARCO_MINILM_L6_GEOMETRY, seed: int = 0) -> np.ndarray:
    """Seeded weights of a classifier geometry: BERT's tensors drawn exactly as :func:`random_blob` draws them (the blob's
    prefix is bit-identical), then the head the same way (sigma 0.02 matrices, zero biases)."""
    return _random_blob(classifier_blob_layout(g), seed)


def load_hf_classifier_state_dict(sd: dict, g: dict | None = None) -> tuple[dict, np.ndarray]:
    """HF ``BertForSequenceClassification`` state dict (``bert.*``, ``bert.pooler.dense.*``, ``classifier.*``) -> (geometry
    with ``num_labels`` from ``classifier.weight``, fp32 blob).  A checkpoint without the pooler (``add_pooling_layer=False``)
    is refused: its logits are not computed from the tanh pooler this runtime applies."""
    if "classifier.weight" not in sd or "classifier.bias" not in sd:
        raise KeyError("no classifier.weight / classifier.bias: a BertForSequenceClassification checkpoint is needed")
    enc = _strip_prefix(sd)
    if "pooler.dense.weight" not in enc or "pooler.dense.bias" not in enc:
        raise ValueError("the checkpoint has no bert.pooler.dense (a model built with add_pooling_layer=False); the classifier "
                         "head here is classifier(tanh(pooler(CLS))) and cannot serve it")
    g, blob = load_hf_state_dict(sd, g)
    cw = _arr(sd["classifier.weight"])
    g["num_labels"] = int(cw.shape[0])
    cb = np.zeros(CLS_B_PAD, np.float32)
    cb[: cw.shape[0]] = _arr(sd["classifier.bias"])
    head = _pack(classifier_blob_layout(g)[len(blob_layout(g)):],
                 {"pool.w": enc["pooler.dense.weight"], "pool.b": enc["pooler.dense.bias"], "cls.w": cw, "cls.b": cb})
    return g, np.concatenate([blob, head])


def load_hf_classifier(sd: dict, cfg: dict) -> tuple[dict, np.ndarray]:
    """A classifier checkpoint's state dict and ``config.json`` (``{}`` without one) -> (geometry with ``num_labels`` and
    ``id2label`` -- the config's, else ``LABEL_i`` --, blob)."""
    g = geometry_from_state_dict(sd, cfg.get("layer_norm_eps", 1e-12), cfg.get("num_attention_heads"))
    g, blob = load_hf_classifier_state_dict(sd, g)
    labels = cfg.get("id2label") or {}
    g["id2label"] = {int(k): str(v) for k, v in labels.items()} if len(labels) == g["num_labels"] else default_id2label(g["num_labels"])
    return g, blob


# ----------------------------------------------------------------------------------------------- SPLADE sparse encoders
# HF BertForMaskedLM checkpoints (naver/splade-v3, naver/splade-cocondenser-ensembledistil, prithivida/Splade_PP_en_v1) that TEI
# serves with --pooling splade through /embed_sparse.  Blob order: blob_layout(g), then mlm.t.w [H,H] | mlm.t.b [H] | mlm.ln.g [H]
# | mlm.ln.b [H] | mlm.dec.w [V,H] | mlm.dec.b [V rounded up to 128] -- the decoder bias padded with zeros, as cls.b is.

MASKED_LM_ARCHITECTURE = "BertForMaskedLM"
_MLM = "cls.predictions."


def splade_blob_layout(g: dict) -> list[tuple[str, tuple[int, ...]]]:
    h, v = g["hidden"], g["vocab"]
    return blob_layout(g) + [("mlm.t.w", (h, h)), ("mlm.t.b", (h,)), ("mlm.ln.g", (h,)), ("mlm.ln.b", (h,)), ("mlm.dec.w", (v, h)),
                             ("mlm.dec.b", ((v + 127) // 128 * 128,))]


def random_splade_blob(g: dict = BGE_BASE_GEOMETRY, seed: int = 0) -> np.ndarray:
    """Seeded weights of a SPLADE geometry: BERT's tensors drawn exactly as :func:`random_blob` draws them (the blob's prefix is
    bit-identical), then the masked-LM head the same way (sigma 0.02 matrices, zero biases, unit LayerNorm; the decoder is not
    tied to the word embeddings)."""
    return _random_blob(splade_blob_layout(g), seed)


def has_masked_lm_head(sd: dict) -> bool:
    return _MLM + "transform.dense.weight" in sd


def load_hf_masked_lm_state_dict(sd: dict, g: dict | None = None) -> tuple[dict, np.ndarray]:
    """HF ``BertForMaskedLM`` state dict (``bert.*`` + ``cls.predictions.*``) -> (geometry, fp32 blob of
    :func:`splade_blob_layout`).  The decoder is ``cls.predictions.decoder.weight``, or the word embeddings when a tied checkpoint
    (safetensors drops the tied copy) leaves it out; its bias is ``cls.predictions.bias`` or ``cls.predictions.decoder.bias``.
    A checkpoint without ``cls.predictions.transform`` is refused: SPLADE's logits come from that head."""
    if not has_masked_lm_head(sd):
        raise ValueError("no cls.predictions.transform.dense.weight: a BertForMaskedLM checkpoint (the masked-LM head SPLADE "
                         "pools) is needed")
    g, blob = load_hf_state_dict(sd, g)
    enc = _strip_prefix(sd)
    dec = sd.get(_MLM + "decoder.weight")
    if dec is None:
        dec = enc["embeddings.word_embeddings.weight"]
    bias = sd.get(_MLM + "bias")
    if bias is None:
        bias = sd.get(_MLM + "decoder.bias")
    if bias is None:
        raise KeyError("no cls.predictions.bias / cls.predictions.decoder.bias")
    head_layout = splade_blob_layout(g)[len(blob_layout(g)):]
    db = np.zeros(head_layout[-1][1], np.float32)
    db[: g["vocab"]] = _arr(bias)
    t = _MLM + "transform."
    head = _pack(head_layout, {"mlm.t.w": sd[t + "dense.weight"], "mlm.t.b": sd[t + "dense.bias"], "mlm.ln.g": sd[t + "LayerNorm.weight"],
                               "mlm.ln.b": sd[t + "LayerNorm.bias"], "mlm.dec.w": dec, "mlm.dec.b": db})
    return g, np.concatenate([blob, head])


def _read_state_dict(path: str) -> dict:
    st = os.path.join(path, "model.safetensors")
    pt = os.path.join(path, "pytorch_model.bin")
    if os.path.exists(st):
        return read_safetensors(st)
    if os.path.exists(pt):
        import torch

        return torch.load(pt, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin under {path}")


def is_masked_lm_dir(path: str) -> bool:
    """Whether a snapshot directory holds a masked-LM checkpoint SPLADE can pool: ``config.json`` names ``BertForMaskedLM``, or
    its weights carry ``cls.predictions.transform``."""
    if MASKED_LM_ARCHITECTURE in hf_architectures(path):
        return True
    try:
        return has_masked_lm_head(_read_state_dict(path))
    except FileNotFoundError:
        return False


def load_hf_masked_lm_dir(path: str) -> tuple[dict, np.ndarray]:
    """A local ``BertForMaskedLM`` snapshot directory -> (geometry, :func:`splade_blob_layout` blob); ``eps`` and the head count
    from its ``config.json``."""
    cfg_path = os.path.join(path, "config.json")
    cfg = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
    sd = _read_state_dict(path)
    return load_hf_masked_lm_state_dict(sd, geometry_from_state_dict(sd, cfg.get("layer_norm_eps", 1e-12), cfg.get("num_attention_heads")))


def resolve_hub_snapshot(cache_dir: str, model_id: str) -> str | None:
    """``<cache>/models--ORG--NAME/snapshots/<rev>/`` as ``huggingface_hub.snapshot_download`` lays it out (the reference
    mounts that cache as a Volume: text_embeddings_inference.py:20-24, 29-34)."""
    root = os.path.join(cache_dir, "models--" + model_id.replace("/", "--"), "snapshots")
    if not os.path.isdir(root):
        return None
    revs = sorted(os.listdir(root))
    return os.path.join(root, revs[-1]) if revs else None


# ----------------------------------------------------------------------------------------------- CLIP ViT image tower
# Second encoder on the same scheduler (SURVEY.md section 8 f3): openai/clip-vit-base-patch16's vision tower as served by the
# reference's image-embedding example (06_gpu_and_ml/embeddings/image_embeddings_infinity.py:76-77, 298-306).
# Blob order (fp32): patch.w [H, 3*p*p] (conv weight flattened channel, row, column) | cls [H] | pos [T, H] | pre.g | pre.b |
# per layer: ln1.g ln1.b qkv.w [3H,H] qkv.b ao.w ao.b ln2.g ln2.b ff1.w [I,H] ff1.b ff2.w [H,I] ff2.b | post.g post.b | proj.w [P, H].

CLIP_VIT_B16_GEOMETRY = dict(image=224, patch=16, hidden=768, layers=12, heads=12, inter=3072, proj=512, eps=1e-5)


def _pre_ln_layer(l: int, h: int, i: int) -> list[tuple[str, tuple[int, ...]]]:
    """One CLIP encoder layer (both towers) in blob order."""
    p = f"l{l}."
    return [(p + "ln1.g", (h,)), (p + "ln1.b", (h,)), (p + "qkv.w", (3 * h, h)), (p + "qkv.b", (3 * h,)),
            (p + "ao.w", (h, h)), (p + "ao.b", (h,)), (p + "ln2.g", (h,)), (p + "ln2.b", (h,)),
            (p + "ff1.w", (i, h)), (p + "ff1.b", (i,)), (p + "ff2.w", (h, i)), (p + "ff2.b", (h,))]


# a CLIP encoder layer's tensors other than Q, K, V: layout name -> HF name under {vision,text}_model.encoder.layers.N.
_CLIP_LAYER = {"ln1.g": "layer_norm1.weight", "ln1.b": "layer_norm1.bias",
               "ao.w": "self_attn.out_proj.weight", "ao.b": "self_attn.out_proj.bias",
               "ln2.g": "layer_norm2.weight", "ln2.b": "layer_norm2.bias",
               "ff1.w": "mlp.fc1.weight", "ff1.b": "mlp.fc1.bias", "ff2.w": "mlp.fc2.weight", "ff2.b": "mlp.fc2.bias"}


def _clip_layers(sd: dict, prefix: str, layers: int) -> dict:
    """``{layout name: tensor}`` of the encoder layers under ``prefix`` (``vision_model.`` / ``text_model.``)."""
    t = {}
    for l in range(layers):
        s, p = f"{prefix}encoder.layers.{l}.", f"l{l}."
        t[p + "qkv.w"] = np.concatenate([_arr(sd[s + f"self_attn.{n}.weight"]) for n in ("q_proj", "k_proj", "v_proj")], 0)
        t[p + "qkv.b"] = np.concatenate([_arr(sd[s + f"self_attn.{n}.bias"]) for n in ("q_proj", "k_proj", "v_proj")], 0)
        t.update({p + name: sd[s + hf] for name, hf in _CLIP_LAYER.items()})
    return t


def vit_blob_layout(g: dict) -> list[tuple[str, tuple[int, ...]]]:
    h, i = g["hidden"], g["inter"]
    tokens = (g["image"] // g["patch"]) ** 2 + 1
    lay = [("patch.w", (h, 3 * g["patch"] * g["patch"])), ("cls", (h,)), ("pos", (tokens, h)), ("pre.g", (h,)), ("pre.b", (h,))]
    for l in range(g["layers"]):
        lay += _pre_ln_layer(l, h, i)
    lay += [("post.g", (h,)), ("post.b", (h,)), ("proj.w", (g["proj"], h))]
    return lay


def vit_blob_numel(g: dict) -> int:
    return sum(int(np.prod(s)) for _, s in vit_blob_layout(g))


def random_vit_blob(g: dict = CLIP_VIT_B16_GEOMETRY, seed: int = 0) -> np.ndarray:
    """Seeded weights of the geometry: normal sigma 0.02 matrices / embeddings, zero biases, unit LayerNorm."""
    return _random_blob(vit_blob_layout(g), seed)


def load_clip_vision_state_dict(sd: dict, eps: float = 1e-5, heads: int | None = None) -> tuple[dict, np.ndarray]:
    """HF ``CLIPModel`` / ``CLIPVisionModelWithProjection`` state dict -> (geometry, fp32 blob).  Parameter names as in HF
    ``modeling_clip.py`` (``vision_model.embeddings.*``, ``vision_model.encoder.layers.N.*``, ``visual_projection.weight``)."""
    pw = _arr(sd["vision_model.embeddings.patch_embedding.weight"])
    h, _, p, _ = pw.shape
    tokens = sd["vision_model.embeddings.position_embedding.weight"].shape[0]
    layers = 0
    while f"vision_model.encoder.layers.{layers}.self_attn.q_proj.weight" in sd:
        layers += 1
    grid = int(round((tokens - 1) ** 0.5))
    g = dict(image=grid * p, patch=int(p), hidden=int(h), layers=layers, heads=int(heads or h // 64),
             inter=int(sd["vision_model.encoder.layers.0.mlp.fc1.weight"].shape[0]), proj=int(sd["visual_projection.weight"].shape[0]), eps=float(eps))
    t = {"patch.w": pw.reshape(h, 3 * p * p), "cls": sd["vision_model.embeddings.class_embedding"],
         "pos": sd["vision_model.embeddings.position_embedding.weight"], "pre.g": sd["vision_model.pre_layrnorm.weight"],
         "pre.b": sd["vision_model.pre_layrnorm.bias"], **_clip_layers(sd, "vision_model.", layers),
         "post.g": sd["vision_model.post_layernorm.weight"], "post.b": sd["vision_model.post_layernorm.bias"],
         "proj.w": sd["visual_projection.weight"]}
    return g, _pack(vit_blob_layout(g), t)


# ----------------------------------------------------------------------------------------------- CLIP text tower
# The other half of the same CLIP checkpoint: openai/clip-vit-base-patch16's (and -patch32's) text tower, which infinity's
# `embed(sentences=...)` runs for the reference's image example (image_embeddings_infinity.py:76-77, 298-306).
# Blob order (fp32): token [V, H] | pos [max_pos, H] | per layer: ln1.g ln1.b qkv.w [3H,H] qkv.b ao.w ao.b ln2.g ln2.b
# ff1.w [I,H] ff1.b ff2.w [H,I] ff2.b | final.g final.b | proj.w [P, H] (text_projection, no bias).
# eos_id: 2 in the original openai configs, which selects HF's legacy pooling (the first position of the largest id).

CLIP_TEXT_B16_GEOMETRY = dict(vocab=49408, hidden=512, layers=12, heads=8, inter=2048, max_pos=77, proj=512, eos_id=2, eps=1e-5)


def clip_text_blob_layout(g: dict) -> list[tuple[str, tuple[int, ...]]]:
    h, i = g["hidden"], g["inter"]
    lay = [("token", (g["vocab"], h)), ("pos", (g["max_pos"], h))]
    for l in range(g["layers"]):
        lay += _pre_ln_layer(l, h, i)
    lay += [("final.g", (h,)), ("final.b", (h,)), ("proj.w", (g["proj"], h))]
    return lay


def clip_text_blob_numel(g: dict) -> int:
    return sum(int(np.prod(s)) for _, s in clip_text_blob_layout(g))


def random_clip_text_blob(g: dict = CLIP_TEXT_B16_GEOMETRY, seed: int = 0) -> np.ndarray:
    """Seeded weights of the geometry: normal sigma 0.02 matrices / embeddings, zero biases, unit LayerNorm."""
    return _random_blob(clip_text_blob_layout(g), seed)


def load_clip_text_state_dict(sd: dict, eps: float = 1e-5, heads: int | None = None, eos_id: int = 2) -> tuple[dict, np.ndarray]:
    """HF ``CLIPModel`` / ``CLIPTextModelWithProjection`` state dict -> (geometry, fp32 blob).  Parameter names as in HF
    ``modeling_clip.py`` (``text_model.embeddings.*``, ``text_model.encoder.layers.N.*``, ``text_model.final_layer_norm``,
    ``text_projection.weight``).  A state dict without ``text_projection.weight`` (a bare ``CLIPTextModel``) is refused: its
    pooled output is not the embedding infinity serves."""
    if "text_projection.weight" not in sd:
        raise KeyError("no text_projection.weight: a CLIPModel or CLIPTextModelWithProjection checkpoint is needed")
    s0 = "text_model."
    vocab, h = sd[s0 + "embeddings.token_embedding.weight"].shape
    layers = 0
    while f"{s0}encoder.layers.{layers}.self_attn.q_proj.weight" in sd:
        layers += 1
    g = dict(vocab=int(vocab), hidden=int(h), layers=layers, heads=int(heads or h // 64),
             inter=int(sd[s0 + "encoder.layers.0.mlp.fc1.weight"].shape[0]),
             max_pos=int(sd[s0 + "embeddings.position_embedding.weight"].shape[0]), proj=int(sd["text_projection.weight"].shape[0]),
             eos_id=int(eos_id), eps=float(eps))
    t = {"token": sd[s0 + "embeddings.token_embedding.weight"], "pos": sd[s0 + "embeddings.position_embedding.weight"],
         **_clip_layers(sd, s0, layers), "final.g": sd[s0 + "final_layer_norm.weight"], "final.b": sd[s0 + "final_layer_norm.bias"],
         "proj.w": sd["text_projection.weight"]}
    return g, _pack(clip_text_blob_layout(g), t)


def clip_text_config_from_dir(path: str) -> dict:
    """(eps, heads, eos_id) of a CLIP snapshot's ``config.json`` ``text_config`` (a CLIPModel) or top level (a
    CLIPTextModelWithProjection); eos_id is 2 -- the original openai configs' value -- when the config does not give it."""
    out = dict(eps=1e-5, heads=None, eos_id=2)
    p = os.path.join(path, "config.json")
    if os.path.exists(p):
        with open(p) as f:
            cfg = json.load(f)
        tc = cfg.get("text_config") or cfg
        out.update(eps=tc.get("layer_norm_eps", 1e-5), heads=tc.get("num_attention_heads"), eos_id=tc.get("eos_token_id", 2))
    return out


# ---- nomic-bert (HF NomicBertModel: nomic-ai/nomic-embed-text-v1 / -v1.5)

NOMIC_ARCHITECTURES = ("NomicBertModel", "NomicBertForPreTraining", "NomicBertForMaskedLM")
NOMIC_MAX_POS = 8192  # the longest input the engine's rotary table and streaming attention take
# nomic-embed-text-v1.5 at its full 8192-token context (rope_theta 1000, mean pooling)
NOMIC_EMBED_TEXT_GEOMETRY = dict(vocab=30528, hidden=768, layers=12, heads=12, inter=3072, max_pos=8192, type_vocab=2, eps=1e-12,
                                 rope_theta=1000.0)


def nomic_blob_layout(g: dict) -> list[tuple[str, tuple[int, ...]]]:
    """HF shapes and order, no biases: word | type | emb.ln, then per layer qkv.w [3H,H] | ao.w | ln1 | gate.w [I,H] | up.w [I,H] |
    down.w [H,I] | ln2."""
    h, i = g["hidden"], g["inter"]
    lay = [("emb.word", (g["vocab"], h)), ("emb.type", (g["type_vocab"], h)), ("emb.ln.g", (h,)), ("emb.ln.b", (h,))]
    for l in range(g["layers"]):
        p = f"l{l}."
        lay += [(p + "qkv.w", (3 * h, h)), (p + "ao.w", (h, h)), (p + "ln1.g", (h,)), (p + "ln1.b", (h,)), (p + "gate.w", (i, h)),
                (p + "up.w", (i, h)), (p + "down.w", (h, i)), (p + "ln2.g", (h,)), (p + "ln2.b", (h,))]
    return lay


def random_nomic_blob(g: dict = NOMIC_EMBED_TEXT_GEOMETRY, seed: int = 0) -> np.ndarray:
    """Seeded weights of a nomic-bert geometry, drawn as :func:`random_blob` draws BERT's (sigma 0.02 matrices and embeddings,
    unit LayerNorm gains, zero offsets), tensor by tensor in :func:`nomic_blob_layout` order."""
    return _random_blob(nomic_blob_layout(g), seed)


def _nomic_names(sd: dict) -> tuple[dict, bool]:
    """Strip a model prefix; True when the keys are the hub checkpoint's (remote-code) names."""
    for pref in ("", "model.", "nomic_bert.", "bert.", "0.auto_model.", "auto_model."):
        if pref + "embeddings.word_embeddings.weight" in sd:
            sd = {k[len(pref):]: v for k, v in sd.items() if k.startswith(pref)}
            return sd, "emb_ln.weight" in sd
    raise KeyError("no nomic-bert weights found (looked for [model.]embeddings.word_embeddings.weight)")


def load_hf_nomic_state_dict(sd: dict, g: dict | None = None) -> tuple[dict, np.ndarray]:
    """A nomic-bert state dict -> (geometry, fp32 blob of :func:`nomic_blob_layout`).  Takes the transformers names
    (``layers.N.self_attn.{q,k,v,o}_proj``, ``layers.N.mlp.{gate,up,down}_proj``, ``layers.N.{post_attention,post_mlp}_layernorm``,
    ``embeddings.LayerNorm``) and the hub checkpoint's (``encoder.layers.N.attn.Wqkv`` = q | k | v on dim 0, ``attn.out_proj``,
    ``mlp.fc12`` = gate, ``mlp.fc11`` = up, ``mlp.fc2`` = down, ``norm1``, ``norm2``, ``emb_ln``); both give the same blob.  ``g``
    (e.g. from :func:`nomic_config_from_dir`) supplies eps, max_pos and rope_theta; the rest is read from the tensors."""
    sd, hub = _nomic_names(sd)
    if hub:
        lp = lambda l: f"encoder.layers.{l}."  # noqa: E731
        names = {"ao.w": "attn.out_proj.weight", "ln1.g": "norm1.weight", "ln1.b": "norm1.bias", "gate.w": "mlp.fc12.weight",
                 "up.w": "mlp.fc11.weight", "down.w": "mlp.fc2.weight", "ln2.g": "norm2.weight", "ln2.b": "norm2.bias"}
        emb_ln = "emb_ln."
    else:
        lp = lambda l: f"layers.{l}."  # noqa: E731
        names = {"ao.w": "self_attn.o_proj.weight", "ln1.g": "post_attention_layernorm.weight", "ln1.b": "post_attention_layernorm.bias",
                 "gate.w": "mlp.gate_proj.weight", "up.w": "mlp.up_proj.weight", "down.w": "mlp.down_proj.weight",
                 "ln2.g": "post_mlp_layernorm.weight", "ln2.b": "post_mlp_layernorm.bias"}
        emb_ln = "embeddings.LayerNorm."
    biases = [k for k in sd if k.endswith(".bias") and "norm" not in k.lower() and not k.startswith("emb_ln")]
    if biases:
        raise ValueError(f"nomic-bert projections carry no bias, but the checkpoint has {biases[0]}")
    layers = 0
    while lp(layers) + names["ao.w"] in sd:
        layers += 1
    vocab, hidden = _arr(sd["embeddings.word_embeddings.weight"]).shape
    base = dict(NOMIC_EMBED_TEXT_GEOMETRY)
    base.update(g or {})
    base.update(vocab=int(vocab), hidden=int(hidden), layers=layers, inter=int(_arr(sd[lp(0) + names["up.w"]]).shape[0]),
                type_vocab=int(_arr(sd["embeddings.token_type_embeddings.weight"]).shape[0]))
    g = base
    t = {"emb.word": sd["embeddings.word_embeddings.weight"], "emb.type": sd["embeddings.token_type_embeddings.weight"],
         "emb.ln.g": sd[emb_ln + "weight"], "emb.ln.b": sd[emb_ln + "bias"]}
    for l in range(layers):
        s, p = lp(l), f"l{l}."
        if hub:
            t[p + "qkv.w"] = sd[s + "attn.Wqkv.weight"]
        else:
            t[p + "qkv.w"] = np.concatenate([_arr(sd[s + f"self_attn.{n}_proj.weight"]) for n in "qkv"], 0)
        t.update({p + name: sd[s + hf] for name, hf in names.items()})
    return g, _pack(nomic_blob_layout(g), t)


def is_nomic_dir(path: str) -> bool:
    """A snapshot whose config.json names NomicBert in ``architectures`` or ``model_type``."""
    p = os.path.join(path, "config.json")
    if not os.path.exists(p):
        return False
    with open(p) as f:
        cfg = json.load(f)
    archs = cfg.get("architectures") or []
    return cfg.get("model_type") == "nomic_bert" or any(a in NOMIC_ARCHITECTURES for a in archs)


def nomic_config_from_dir(path: str) -> dict:
    """The geometry of a nomic-bert snapshot's config.json.  Reads the transformers field names (``hidden_size``,
    ``num_attention_heads``, ``intermediate_size``, ``num_hidden_layers``, ``max_position_embeddings``, ``layer_norm_eps``,
    ``rope_parameters.rope_theta`` / ``rope_type``) or the remote-code ones (``n_embd``, ``n_head``, ``n_inner``, ``n_layer``,
    ``layer_norm_epsilon``, ``rotary_emb_base``, ``max_trained_positions``).  Refuses, with a message, what the engine does not
    compute: another rope_type, ``rotary_scaling_factor`` (dynamic NTK), interleaved or partial rotary, pre-norm, biases, and any
    activation but SwiGLU.  max_pos is ``max_position_embeddings``, else ``max_trained_positions``, else 2048, at most 8192."""
    with open(os.path.join(path, "config.json")) as f:
        cfg = json.load(f)
    return nomic_config(cfg)


def nomic_config(cfg: dict) -> dict:
    """:func:`nomic_config_from_dir` on a parsed config.json."""
    def pick(*names, default=None):
        for n in names:
            if cfg.get(n) is not None:
                return cfg[n]
        return default

    rope = cfg.get("rope_parameters") or {}
    rope_type = rope.get("rope_type", cfg.get("rope_type", "default"))
    if rope_type != "default":
        raise ValueError(f"rope_type {rope_type!r} is not supported (only 'default' rotary embeddings)")
    if cfg.get("rotary_scaling_factor") is not None:
        raise ValueError("rotary_scaling_factor (dynamic-NTK context extension) is not supported")
    if cfg.get("rotary_emb_interleaved"):
        raise ValueError("rotary_emb_interleaved: true is not supported (rotate_half pairs (d, d + 32) only)")
    if float(cfg.get("rotary_emb_fraction", 1.0)) != 1.0:
        raise ValueError(f"rotary_emb_fraction {cfg['rotary_emb_fraction']} is not supported (every head dimension rotates)")
    if cfg.get("prenorm"):
        raise ValueError("prenorm: true is not supported (nomic-bert layers are post-LayerNorm)")
    on = [k for k, v in cfg.items() if k.endswith("_bias") and v is True]
    if on:
        raise ValueError(f"{on[0]}: true is not supported (nomic-bert projections carry no bias)")
    act = pick("activation_function", "hidden_act", default="swiglu")
    if act not in ("swiglu", "silu"):
        raise ValueError(f"activation {act!r} is not supported (SwiGLU only)")
    max_pos = pick("max_position_embeddings", "max_trained_positions", default=2048)
    theta = rope.get("rope_theta", pick("rotary_emb_base", "rope_theta", default=1000.0))
    return dict(vocab=int(pick("vocab_size", default=30528)), hidden=int(pick("hidden_size", "n_embd", default=768)),
                layers=int(pick("num_hidden_layers", "n_layer", default=12)), heads=int(pick("num_attention_heads", "n_head", default=12)),
                inter=int(pick("intermediate_size", "n_inner", default=3072)), max_pos=min(int(max_pos), NOMIC_MAX_POS),
                type_vocab=int(pick("type_vocab_size", default=2)), eps=float(pick("layer_norm_eps", "layer_norm_epsilon", default=1e-12)),
                rope_theta=float(theta))


def load_hf_nomic_dir(path: str) -> tuple[dict, np.ndarray]:
    """A nomic-bert snapshot directory -> (geometry, blob)."""
    return load_hf_nomic_state_dict(_read_state_dict(path), nomic_config_from_dir(path))
