"""In-box stand-in for the ``infinity_emb`` engine API that the reference's image-embedding example drives
(06_gpu_and_ml/embeddings/image_embeddings_infinity.py:126-127, 296-306, 340-356): ``AsyncEmbeddingEngine.from_args(
EngineArgs(model_name_or_path="openai/clip-vit-base-patch16", engine=torch, dtype=float16, device="cuda"))``,
``await engine.astart()``, ``embeddings, usage = await engine.image_embed(images=[PIL images])``, ``await engine.astop()``.

Like ``text-embeddings-router`` (tei_router/), it is the boundary the reference script already talks to, re-implemented
over the b200rt C ABI: the CLIP ViT-B/16 image tower runs on the hand-written sm_90a kernels (kind "vit"), preprocessing
is preprocess.clip_preprocess.  The reference starts one engine per concurrent input to pack a GPU with model copies
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
_models: dict[str, dict] = {}  # model name -> {"model": ImageEmbedModel, "refs": n}
_runtime_refs = 0
_owns_runtime = False  # whether the first engine brought the runtime up (then the last one shuts it down)


def _load_clip(args: EngineArgs):
    """(geometry, blob, source) for ``args.model_name_or_path``: an explicit weights file / HF directory, else the hub
    snapshot under $HF_HOME/hub (the reference points HF_HOME at its volume, :112-117), else seeded random init."""
    import numpy as np
    from b200rt import weights as W

    def from_dir(d):
        for name in ("model.safetensors", "pytorch_model.bin"):
            p = os.path.join(d, name)
            if os.path.exists(p):
                if name.endswith(".safetensors"):
                    sd = W.read_safetensors(p)
                else:
                    import torch

                    sd = {k: v.float().numpy() for k, v in torch.load(p, map_location="cpu", weights_only=True).items()}
                return W.load_clip_vision_state_dict(sd) + (p,)
        return None

    cand = args.weights or args.model_name_or_path
    if cand.endswith(".safetensors") and os.path.exists(cand):
        return W.load_clip_vision_state_dict(W.read_safetensors(cand)) + (cand,)
    if os.path.isdir(cand):
        got = from_dir(cand)
        if got:
            return got
    if args.weights and os.path.isfile(args.weights):
        return dict(W.CLIP_VIT_B16_GEOMETRY), np.fromfile(args.weights, np.float32), args.weights
    for root in (os.environ.get("HF_HUB_CACHE"), os.path.join(os.environ.get("HF_HOME", ""), "hub") if os.environ.get("HF_HOME") else None):
        if root and os.path.isdir(root):
            snap = W.resolve_hub_snapshot(root, args.model_name_or_path)
            got = from_dir(snap) if snap else None
            if got:
                return got
    return dict(W.CLIP_VIT_B16_GEOMETRY), W.random_vit_blob(W.CLIP_VIT_B16_GEOMETRY), None


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
        return {"image_embed"}

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
                    geometry, blob, source = _load_clip(a)
                    if source is None:
                        print(f"[infinity_emb/b200] no weights for {a.model_name_or_path!r} offline: seeded random init", file=sys.stderr)
                    else:
                        print(f"[infinity_emb/b200] weights: {source}", file=sys.stderr)
                    e = _models[a.model_name_or_path] = {"model": b200rt.ImageEmbedModel(geometry, blob), "refs": 0, "image": geometry["image"]}
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

    async def embed(self, *, sentences):
        raise NotImplementedError("infinity_emb/b200rt serves the image tower only; text goes through text-embeddings-router (tei_router)")


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
