"""In-box stand-in for the ``infinity_emb`` engine API that the reference's image-embedding example drives
(06_gpu_and_ml/embeddings/image_embeddings_infinity.py:126-127, 296-306, 340-356): ``AsyncEmbeddingEngine.from_args(
EngineArgs(model_name_or_path="openai/clip-vit-base-patch16", engine=torch, dtype=float16, device="cuda"))``,
``await engine.astart()``, ``embeddings, usage = await engine.image_embed(images=[PIL images])``, ``await engine.astop()``
-- and, for searching those images with text, ``embeddings, usage = await engine.embed(sentences=[...])``.

Like ``text-embeddings-router`` (tei_router/), it is the boundary the reference script already talks to, re-implemented
over the b200rt C ABI: both towers of the CLIP model run on the hand-written sm_90a kernels -- the ViT-B/16 image tower
(kind "vit", preprocessing by preprocess.clip_preprocess) and the text tower (kind "clip_text", tokenisation by
clip_tokenizer, CLIP's byte-level BPE) -- loaded from the same checkpoint, so ``100 cos(image, text)`` is CLIP's
``logits_per_image``.  The reference starts one engine per concurrent input to pack a GPU with model copies
(``n_engines``, :283-306); here every engine object of a process shares ONE loaded model and the scheduler's replica pool --
concurrency comes from tickets in flight, not from model copies.  There is no CPU path: without the CUDA library (or a
GPU) ``astart`` raises.
"""
from __future__ import annotations

import asyncio
import dataclasses
import os
import sys
import threading

from .primitives import Device, Dtype, InferenceEngine

__version__ = "0.0.76+b200rt"
__all__ = ["AsyncEmbeddingEngine", "AsyncEngineArray", "EngineArgs"]


@dataclasses.dataclass
class EngineArgs:
    model_name_or_path: str = "openai/clip-vit-base-patch16"
    batch_size: int = 32
    revision: str | None = None
    trust_remote_code: bool = True
    engine: InferenceEngine = InferenceEngine.torch
    model_warmup: bool = False
    vector_disk_cache_path: str = ""
    device: str | Device = "cuda"
    device_id: object = None
    compile: bool = False
    bettertransformer: bool = True
    dtype: Dtype | str = Dtype.auto
    pooling_method: str = "auto"
    lengths_via_tokenize: bool = False
    embedding_dtype: str = "float32"
    served_model_name: str | None = None
    # b200rt-specific (the reference never sets them): GPUs for the replica pool (0 = all visible), explicit weights
    n_gpus: int = 0
    weights: str = ""


_lock = threading.Lock()
_models: dict[str, dict] = {}  # model name -> {"model": ImageEmbedModel, "text": ClipTextModel, "tok": ClipTokenizer, "refs": n}
_runtime_refs = 0
_owns_runtime = False  # whether the first engine brought the runtime up (then the last one shuts it down)


def _towers(sd: dict, cfg_dir: str):
    """(vision (geometry, blob), text (geometry, blob) or None) of one CLIPModel state dict; the text tower's eps, heads and
    eos_token_id come from the snapshot's config.json (``text_config``) when there is one."""
    from b200rt import weights as W

    text = None
    if "text_projection.weight" in sd and "text_model.embeddings.token_embedding.weight" in sd:
        text = W.load_clip_text_state_dict(sd, **W.clip_text_config_from_dir(cfg_dir))
    return W.load_clip_vision_state_dict(sd), text


def _load_clip(args: EngineArgs) -> dict:
    """Both towers of ``args.model_name_or_path`` from one source: an explicit weights file / HF directory, else the hub
    snapshot under $HF_HOME/hub (the reference points HF_HOME at its volume, :112-117), else seeded random init.  Returns
    dict(vision=(geometry, blob), text=(geometry, blob) or None when the source holds no text tower, source=path or None,
    tok_dir=the directory holding vocab.json / merges.txt, if any)."""
    import numpy as np
    from b200rt import weights as W

    def from_file(p):
        if p.endswith(".safetensors"):
            sd = W.read_safetensors(p)
        else:
            import torch

            sd = {k: v.float().numpy() for k, v in torch.load(p, map_location="cpu", weights_only=True).items()}
        d = os.path.dirname(os.path.abspath(p))
        vision, text = _towers(sd, d)
        return dict(vision=vision, text=text, source=p, tok_dir=d)

    def from_dir(d):
        for name in ("model.safetensors", "pytorch_model.bin"):
            p = os.path.join(d, name)
            if os.path.exists(p):
                return from_file(p)
        return None

    cand = args.weights or args.model_name_or_path
    if cand.endswith(".safetensors") and os.path.exists(cand):
        return from_file(cand)
    if os.path.isdir(cand):
        got = from_dir(cand)
        if got:
            return got
    if args.weights and os.path.isfile(args.weights):
        return dict(vision=(dict(W.CLIP_VIT_B16_GEOMETRY), np.fromfile(args.weights, np.float32)), text=None, source=args.weights, tok_dir=None)
    for root in (os.environ.get("HF_HUB_CACHE"), os.path.join(os.environ.get("HF_HOME", ""), "hub") if os.environ.get("HF_HOME") else None):
        if root and os.path.isdir(root):
            snap = W.resolve_hub_snapshot(root, args.model_name_or_path)
            got = from_dir(snap) if snap else None
            if got:
                return got
    return dict(vision=(dict(W.CLIP_VIT_B16_GEOMETRY), W.random_vit_blob(W.CLIP_VIT_B16_GEOMETRY)), text=None, source=None, tok_dir=None)


class AsyncEmbeddingEngine:
    def __init__(self, args: EngineArgs):
        self._args = args
        self._entry = None
        self.running = False

    @classmethod
    def from_args(cls, engine_args: EngineArgs) -> "AsyncEmbeddingEngine":
        return cls(engine_args)

    @property
    def engine_args(self) -> EngineArgs:
        return self._args

    @property
    def capabilities(self) -> set:
        return {"embed", "image_embed"}

    def _start(self):
        global _runtime_refs, _owns_runtime
        import b200rt

        a = self._args
        dev = a.device.value if isinstance(a.device, Device) else str(a.device)
        if dev not in ("cuda", "auto"):
            raise ValueError(f"infinity_emb/b200rt: device={dev!r} is not available: the engine runs on H100 GPUs only")
        with _lock:
            if _runtime_refs == 0:
                _owns_runtime = not b200rt._initialised  # an application may already run the pool for its text models
                if _owns_runtime:
                    n = a.n_gpus
                    if n <= 0:
                        import torch

                        n = max(1, torch.cuda.device_count())
                    b200rt.init(n)
            _runtime_refs += 1
            try:
                e = _models.get(a.model_name_or_path)
                if e is None:
                    from b200rt import weights as W

                    from .clip_tokenizer import ClipTokenizer

                    got = _load_clip(a)
                    if got["source"] is None:
                        print(f"[infinity_emb/b200] no weights for {a.model_name_or_path!r} offline: seeded random init", file=sys.stderr)
                    else:
                        print(f"[infinity_emb/b200] weights: {got['source']}", file=sys.stderr)
                    vg, vblob = got["vision"]
                    tg, tblob = got["text"] or (dict(W.CLIP_TEXT_B16_GEOMETRY), W.random_clip_text_blob(W.CLIP_TEXT_B16_GEOMETRY))
                    if got["text"] is None and got["source"] is not None:
                        print(f"[infinity_emb/b200] {got['source']} holds no text tower: the text tower is seeded random init", file=sys.stderr)
                    tok = ClipTokenizer.from_dir(got["tok_dir"])
                    if tok.synthetic:
                        print("[infinity_emb/b200] ********************************************************************\n"
                              "[infinity_emb/b200] NO CLIP vocab.json / merges.txt next to the weights: sentences are tokenised with\n"
                              "[infinity_emb/b200] CLIP's merge-free base vocabulary (one token per byte).  Text embeddings are NOT\n"
                              "[infinity_emb/b200] the real model's; token-id inputs are unaffected.\n"
                              "[infinity_emb/b200] ********************************************************************", file=sys.stderr)
                    e = _models[a.model_name_or_path] = {"model": b200rt.ImageEmbedModel(vg, vblob), "text": b200rt.ClipTextModel(tg, tblob),
                                                         "tok": tok, "refs": 0, "image": vg["image"]}
            except BaseException:  # a failed load must not leave the runtime referenced by an engine that never ran
                _runtime_refs -= 1
                if _runtime_refs == 0 and _owns_runtime:
                    b200rt.shutdown()
                raise
            e["refs"] += 1
            self._entry = e
            self.running = True

    def _stop(self):
        global _runtime_refs
        import b200rt

        with _lock:
            if not self.running:
                return
            self.running = False
            self._entry["refs"] -= 1
            if self._entry["refs"] == 0:
                _models.pop(self._args.model_name_or_path, None)
            self._entry = None
            _runtime_refs -= 1
            if _runtime_refs == 0 and _owns_runtime:
                b200rt.shutdown()

    async def astart(self):
        await asyncio.get_running_loop().run_in_executor(None, self._start)

    async def astop(self):
        await asyncio.get_running_loop().run_in_executor(None, self._stop)

    async def __aenter__(self):
        await self.astart()
        return self

    async def __aexit__(self, *exc):
        await self.astop()

    def _image_embed(self, images):
        from .preprocess import clip_preprocess

        if not self.running:
            raise RuntimeError("engine is not running: call `await engine.astart()` first")
        e = self._entry
        pixels = clip_preprocess(images, e["image"])
        out = e["model"].embed(pixels)  # [n, proj] float32, unit norm; blocks in b200rt_wait with the GIL released
        return list(out), len(images)

    async def image_embed(self, *, images):
        """``(embeddings, usage)``: one unit-norm float32 vector per image (PIL images or uint8 arrays)."""
        if len(images) == 0:
            return [], 0
        return await asyncio.get_running_loop().run_in_executor(None, self._image_embed, list(images))

    def _embed(self, sentences):
        if not self.running:
            raise RuntimeError("engine is not running: call `await engine.astart()` first")
        e = self._entry
        ids, lens = e["tok"].batch(sentences)
        out = e["text"].embed(ids, lens)  # [n, proj] float32, unit norm, in the image tower's space
        return list(out), int(lens.sum())

    async def embed(self, *, sentences):
        """``(embeddings, usage)``: one unit-norm float32 vector per sentence, in the image embeddings' space (CLIP's text
        tower); usage is the number of tokens, start and end tokens included."""
        if len(sentences) == 0:
            return [], 0
        return await asyncio.get_running_loop().run_in_executor(None, self._embed, list(sentences))


class AsyncEngineArray:
    """``AsyncEngineArray.from_args([EngineArgs, ...])`` -> indexable by model name (infinity_emb's multi-model front)."""

    def __init__(self, engines):
        self._engines = {e.engine_args.served_model_name or e.engine_args.model_name_or_path: e for e in engines}

    @classmethod
    def from_args(cls, engine_args_array):
        return cls([AsyncEmbeddingEngine.from_args(a) for a in engine_args_array])

    def __iter__(self):
        return iter(self._engines.values())

    def __getitem__(self, name):
        return self._engines[name]

    async def astart(self):
        for e in self:
            await e.astart()

    async def astop(self):
        for e in self:
            await e.astop()
