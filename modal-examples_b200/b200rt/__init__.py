"""ctypes binding of ``libb200rt.so`` (C ABI in ``include/b200rt.h``).

This is the host-side mirror of the reference's interface for the embed hot path: where the
reference's ``TextEmbeddingsInference.embed`` (``06_gpu_and_ml/embeddings/text_embeddings_inference.py:97-104``)
POSTs strings to a TEI server and ``.map`` (``:167``) fans batches out to cloud containers, an
:class:`EmbedModel` takes token-id batches and the library's C++ scheduler fans them out to the local
H100s.  There is no CPU path: importing works anywhere, but :func:`init` raises unless the shared
library is built and an H100 is visible.
"""
from __future__ import annotations

import ctypes
import os
import threading
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libb200rt.so")

OK, TIMEOUT = 0, 1
E_INVALID, E_STATE, E_CUDA, E_NOMEM, E_UNSUPPORTED = -1, -2, -3, -4, -5

# every symbol include/b200rt.h and include/b200rt_debug.h declare (tests check the export list)
ABI_SYMBOLS = [
    "b200rt_init", "b200rt_init_devices", "b200rt_num_gpus", "b200rt_model_load", "b200rt_model_load_ex", "b200rt_submit", "b200rt_submit_ex", "b200rt_submit_pixels", "b200rt_wait",
    "b200rt_poll_any", "b200rt_embed_device", "b200rt_device_sync", "b200rt_submit_pairs", "b200rt_embed_device_pairs", "b200rt_wave_capacity_items", "b200rt_model_wave_capacity_items",
    "b200rt_alloc_pinned", "b200rt_free_pinned", "b200rt_stats", "b200rt_last_error", "b200rt_shutdown",
]
DEBUG_SYMBOLS = ["b200rt_debug_gemm", "b200rt_debug_gemm_ex", "b200rt_debug_attention", "b200rt_debug_attention_ex", "b200rt_debug_profile_forward",
                 "b200rt_debug_embed", "b200rt_debug_vit_embed", "b200rt_debug_pool_normalize", "b200rt_debug_mean_pool_normalize",
                 "b200rt_debug_vit_pool", "b200rt_debug_clip_text_pool", "b200rt_debug_fold_ln",
                 "b200rt_debug_forward_trace", "b200rt_debug_vit_forward_trace", "b200rt_debug_model_cap_rows",
                 "b200rt_debug_embed_segs", "b200rt_debug_cls_head", "b200rt_debug_forward_trace_segs",
                 "b200rt_debug_gemm_splade", "b200rt_debug_mlm_ln_stats", "b200rt_debug_splade_finalize",
                 "b200rt_debug_gemm_rope", "b200rt_debug_gemm_swiglu", "b200rt_debug_attention_stream"]


def SPLIT_SMS(k: int) -> int:
    """``init`` flag (B200RT_INIT_SPLIT_SMS): two replicas per GPU, each replica's GEMMs on all but k SMs, its attention on k."""
    return (k & 0xFF) << 16


class B200RTError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200rt error {code}: {msg}")
        self.code = code


class BertConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("vocab", "hidden", "layers", "heads", "inter", "max_pos", "type_vocab")] + [
        ("eps", ctypes.c_float)
    ]


class BertClassifierConfig(ctypes.Structure):
    _fields_ = [("bert", BertConfig), ("num_labels", ctypes.c_int32)]


class NomicBertConfig(ctypes.Structure):
    _fields_ = [("bert", BertConfig), ("rope_theta", ctypes.c_float)]


class VitConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("image", "patch", "hidden", "layers", "heads", "inter", "proj")] + [("eps", ctypes.c_float)]


class ClipTextConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("vocab", "hidden", "layers", "heads", "inter", "max_pos", "proj", "eos_id")] + [
        ("eps", ctypes.c_float)
    ]


class Stats(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in ("items", "waves", "tickets", "kernel_launches", "h2d_bytes", "d2h_bytes", "peer_bytes")] + [
        (n, ctypes.c_double) for n in ("stage_us", "h2d_scatter_us", "forward_us", "d2h_us", "gap_us", "dispatch_us", "forward_max_us", "gap_max_us")
    ]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


_lib = None
_lib_lock = threading.Lock()


def load_library():
    """dlopen the C ABI.  Fails loudly when the extension has not been built."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise B200RTError(E_STATE, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                       "(there is no CPU or PyTorch fallback for this path)")
        lib = ctypes.CDLL(LIB_PATH)
        i32p = ctypes.POINTER(ctypes.c_int32)
        f32p = ctypes.POINTER(ctypes.c_float)
        u16p = ctypes.POINTER(ctypes.c_uint16)
        u64p = ctypes.POINTER(ctypes.c_uint64)
        lib.b200rt_init.argtypes = [ctypes.c_int, ctypes.c_uint32]
        lib.b200rt_init_devices.argtypes = [i32p, ctypes.c_int, ctypes.c_uint32]
        lib.b200rt_model_load.argtypes = [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, i32p]
        lib.b200rt_model_load_ex.argtypes = [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, i32p]
        lib.b200rt_submit.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, u64p]
        lib.b200rt_submit_ex.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.c_uint32, u64p]
        lib.b200rt_submit_pixels.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, u64p]
        lib.b200rt_submit_pairs.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_void_p, ctypes.c_uint32, u64p]
        lib.b200rt_wait.argtypes = [ctypes.c_uint64, ctypes.c_int]
        lib.b200rt_poll_any.argtypes = [u64p, ctypes.c_int]
        lib.b200rt_embed_device.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        lib.b200rt_embed_device_pairs.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_int,
                                                                                                      ctypes.c_void_p, ctypes.c_void_p]
        lib.b200rt_device_sync.argtypes = [ctypes.c_int]
        lib.b200rt_model_wave_capacity_items.argtypes = [ctypes.c_int]
        lib.b200rt_debug_model_cap_rows.argtypes = [ctypes.c_int]
        lib.b200rt_alloc_pinned.argtypes = [ctypes.c_size_t]
        lib.b200rt_alloc_pinned.restype = ctypes.c_void_p
        lib.b200rt_free_pinned.argtypes = [ctypes.c_void_p]
        lib.b200rt_free_pinned.restype = None
        lib.b200rt_stats.argtypes = [ctypes.POINTER(Stats)]
        lib.b200rt_last_error.restype = ctypes.c_char_p
        lib.b200rt_shutdown.restype = None
        lib.b200rt_debug_gemm.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, f32p, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_int,
                                          ctypes.POINTER(ctypes.c_int)]
        lib.b200rt_debug_gemm_ex.argtypes = lib.b200rt_debug_gemm.argtypes + [ctypes.c_uint32]
        lib.b200rt_debug_attention.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, f32p,
                                               ctypes.c_int, ctypes.c_int, ctypes.c_int]
        lib.b200rt_debug_attention_ex.argtypes = lib.b200rt_debug_attention.argtypes + [ctypes.c_uint32]
        vp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        lib.b200rt_debug_embed.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp, vp, vp, ci]
        lib.b200rt_debug_vit_embed.argtypes = [vp, vp, vp, vp, vp, ci, ci, cf, vp, vp, vp]
        lib.b200rt_debug_embed_segs.argtypes = [vp] * 5 + [ci, ci, ci, vp, vp, vp, ci]
        lib.b200rt_debug_cls_head.argtypes = [vp] * 8 + [ci, ci, ci, cf, vp, ci, ci]
        lib.b200rt_debug_pool_normalize.argtypes = [vp, vp, vp, vp, ci, ci, cf, vp, ci]
        lib.b200rt_debug_mean_pool_normalize.argtypes = [vp, vp, vp, vp, vp, ci, ci, cf, vp, ci]
        lib.b200rt_debug_vit_pool.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, cf, vp]
        lib.b200rt_debug_clip_text_pool.argtypes = [vp] * 7 + [ci, ci, ci, cf, ci, vp]
        lib.b200rt_debug_fold_ln.argtypes = [vp, vp, vp, vp, ci, ci, vp, vp]
        lib.b200rt_debug_forward_trace.argtypes = [ci, vp, vp, ci, ci, ci] + [vp] * 8 + [ctypes.c_char_p, ctypes.c_size_t, i32p]
        lib.b200rt_debug_vit_forward_trace.argtypes = [ci, vp, ci, ci] + [vp] * 8 + [ctypes.c_char_p, ctypes.c_size_t, i32p]
        lib.b200rt_debug_forward_trace_segs.argtypes = [ci, vp, vp, vp, ci, ci, ci] + [vp] * 8 + [ctypes.c_char_p, ctypes.c_size_t, i32p]
        lib.b200rt_debug_gemm_splade.argtypes = [vp] * 5 + [ci] * 5 + [cf, ci, ci, f32p, vp, i32p]
        lib.b200rt_debug_mlm_ln_stats.argtypes = [vp, ci, ci, ctypes.c_size_t, vp, vp]
        lib.b200rt_debug_splade_finalize.argtypes = [vp, ci, ci, ci, vp]
        lib.b200rt_debug_gemm_rope.argtypes = [vp] * 5 + [ci] * 5 + [cf, ci, vp, i32p]
        lib.b200rt_debug_gemm_swiglu.argtypes = [vp] * 4 + [ci, ci, cf, ci, vp, i32p]
        lib.b200rt_debug_attention_stream.argtypes = [vp, vp, ci, ci, vp, ci, ci, f32p]
        lib.b200rt_debug_profile_forward.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t,
                                                     f32p, i32p, ctypes.c_int]
        _lib = lib
        return lib


def _check(rc: int):
    if rc < 0:
        raise B200RTError(rc, (load_library().b200rt_last_error() or b"").decode(errors="replace"))
    return rc


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


# --------------------------------------------------------------------------------------------- runtime

_initialised = False


def init(n_gpus: int = 1, devices=None, flags: int = 0, wave_items: int = 0) -> int:
    """Start the replica pool on ``devices`` (default ``0..n_gpus-1``).  Idempotent per process.
    ``wave_items``: 512-token items one replica takes per wave (0 = the library default: one per SM, 132 on an H100 SXM)."""
    global _initialised
    lib = load_library()
    if _initialised:
        return lib.b200rt_num_gpus()
    flags |= wave_items & 0xFFFF
    if devices is not None:
        arr = (ctypes.c_int32 * len(devices))(*devices)
        _check(lib.b200rt_init_devices(arr, len(devices), flags))
    else:
        _check(lib.b200rt_init(n_gpus, flags))
    _initialised = True
    return lib.b200rt_num_gpus()


def shutdown():
    global _initialised
    if _initialised:
        load_library().b200rt_shutdown()
        _initialised = False


def num_gpus() -> int:
    return _check(load_library().b200rt_num_gpus())


def wave_capacity_items() -> int:
    """Items of 512 tokens one replica takes per wave of a bge-base or bge-small model (see EmbedModel.wave_capacity_items)."""
    return _check(load_library().b200rt_wave_capacity_items())


def stats() -> dict:
    s = Stats()
    _check(load_library().b200rt_stats(ctypes.byref(s)))
    return s.as_dict()


class PinnedBuffer:
    """Page-locked host array (``b200rt_alloc_pinned``)."""

    def __init__(self, shape, dtype):
        self.shape = tuple(int(x) for x in np.atleast_1d(shape))
        self.dtype = np.dtype(dtype)
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        self._p = load_library().b200rt_alloc_pinned(max(nbytes, 1))
        if not self._p:
            _check(E_NOMEM)
        buf = (ctypes.c_char * nbytes).from_address(self._p)
        self.array = np.frombuffer(buf, dtype=self.dtype).reshape(self.shape)

    def free(self):
        if self._p:
            self.array = None
            load_library().b200rt_free_pinned(self._p)
            self._p = None


@dataclass
class Ticket:
    id: int
    out: np.ndarray
    tag: object = None
    ids: object = None  # keeps a lent (BORROW_IDS) input alive until the ticket completes


class TicketError(B200RTError):
    """A ticket completed with an error; carries the ticket so that the caller can tell which input failed."""

    def __init__(self, code: int, msg: str, ticket: "Ticket | None"):
        super().__init__(code, msg)
        self.ticket = ticket


# b200rt_poll_any is process-global, so the registry of live tickets is too (not per model): a ticket is registered
# under the lock that also covers its b200rt_submit call, so a poll_any thread that reaps it early blocks on the lock
# until the entry exists.
_live: dict[int, Ticket] = {}
_live_lock = threading.Lock()

SUBMIT_BORROW_IDS = 1


def poll_any(timeout_ms: int = -1) -> Ticket | None:
    """Next finished ticket nobody is waiting on (any model); None on timeout.  Raises :class:`TicketError` (with the
    ticket attached) when that ticket failed."""
    lib = load_library()
    t = ctypes.c_uint64(0)
    rc = lib.b200rt_poll_any(ctypes.byref(t), timeout_ms)
    if rc == TIMEOUT:
        return None
    with _live_lock:
        tk = _live.pop(t.value, None)
    if rc < 0:
        msg = (lib.b200rt_last_error() or b"").decode(errors="replace")
        if t.value == 0:
            raise B200RTError(rc, msg)
        raise TicketError(rc, msg, tk)
    return tk


LOAD_POOL_MEAN = 1
POOLINGS = ("cls", "mean")


def _pool_flags(pooling: str) -> int:
    """The load flags of a text encoder's ``pooling``."""
    if pooling not in POOLINGS:
        raise B200RTError(E_INVALID, f"pooling must be one of {POOLINGS}, got {pooling!r}")
    return LOAD_POOL_MEAN if pooling == "mean" else 0


def _load(model, kind: bytes, cfg, blob: np.ndarray, flags: int = 0):
    """b200rt_model_load_ex of ``blob`` as a model of ``kind``; gives ``model`` its ``cfg``, ``handle`` and the library it calls."""
    lib = load_library()
    blob = np.ascontiguousarray(blob, dtype=np.float32)
    h = ctypes.c_int32(-1)
    _check(lib.b200rt_model_load_ex(kind, ctypes.byref(cfg), _ptr(blob), blob.nbytes, flags, ctypes.byref(h)))
    model.cfg, model.handle, model._lib = cfg, h.value, lib


def _bert_config(g: dict) -> BertConfig:
    return BertConfig(g["vocab"], g["hidden"], g["layers"], g["heads"], g["inter"], g["max_pos"], g["type_vocab"], g["eps"])


class EmbedModel:
    """A loaded BERT-geometry encoder; ``submit``/``wait``/``poll_any`` are the .map() primitives.
    ``pooling``: "cls" (the [CLS] row: bge) or "mean" (the mean of the valid tokens' final hidden states, as
    sentence-transformers' Pooling(mean) computes it: all-MiniLM-L6-v2, e5, gte); either way the result is L2-normalised."""

    def __init__(self, geometry: dict, blob: np.ndarray, pooling: str = "cls"):
        g = geometry
        self.hidden, self.inter = g["hidden"], g["inter"]
        self.out_dim = self.hidden
        self.pooling = pooling
        _load(self, b"bert", _bert_config(g), blob, _pool_flags(pooling))

    def submit(self, ids: np.ndarray, lens=None, out: np.ndarray | None = None, tag=None, borrow_ids: bool = False) -> Ticket:
        """``borrow_ids``: the caller promises not to touch ``ids`` until the ticket completes; the library then takes
        no private copy and, when ``ids``/``out`` live in :class:`PinnedBuffer` memory, DMAs from/to them directly."""
        return self._submit(ids, lens, None, out, tag, borrow_ids)

    def _submit(self, ids, lens, segs, out, tag, borrow_ids) -> Ticket:
        """b200rt_submit_ex, or b200rt_submit_pairs when ``segs`` (int32 [n_items]) is given."""
        if borrow_ids and not (isinstance(ids, np.ndarray) and ids.dtype == np.int32 and ids.flags.c_contiguous):
            raise B200RTError(E_INVALID, "borrow_ids needs a C-contiguous int32 array (a converted copy would be freed too early)")
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        if ids.ndim != 2:
            raise B200RTError(E_INVALID, f"ids must be [n_items, max_len], got shape {ids.shape}")
        n, S = ids.shape
        if lens is not None:
            lens = np.ascontiguousarray(lens, dtype=np.int32)
            if lens.shape != (n,):
                raise B200RTError(E_INVALID, f"lens must have shape ({n},), got {lens.shape}")
        if out is None:
            out = np.empty((n, self.out_dim), np.float32)
        elif out.dtype != np.float32 or not out.flags.c_contiguous or out.shape != (n, self.out_dim):
            raise B200RTError(E_INVALID, f"out must be a C-contiguous float32 [n_items, {self.out_dim}] array")
        if segs is not None:
            segs = np.ascontiguousarray(segs, dtype=np.int32)
            if segs.shape != (n,):
                raise B200RTError(E_INVALID, f"segs must have shape ({n},), got {segs.shape}")
        t = ctypes.c_uint64(0)
        flags = SUBMIT_BORROW_IDS if borrow_ids else 0
        lens_p = _ptr(lens) if lens is not None else None
        with _live_lock:
            if segs is None:
                _check(self._lib.b200rt_submit_ex(self.handle, _ptr(ids), lens_p, n, S, _ptr(out), flags, ctypes.byref(t)))
            else:
                _check(self._lib.b200rt_submit_pairs(self.handle, _ptr(ids), lens_p, _ptr(segs), n, S, _ptr(out), flags, ctypes.byref(t)))
            tk = Ticket(t.value, out, tag, ids if borrow_ids else None)
            _live[tk.id] = tk
        return tk

    def wait(self, ticket: Ticket, timeout_ms: int = -1) -> np.ndarray | None:
        rc = self._lib.b200rt_wait(ticket.id, timeout_ms)
        if rc == TIMEOUT:
            return None
        with _live_lock:
            _live.pop(ticket.id, None)
        if rc < 0:
            raise TicketError(rc, (self._lib.b200rt_last_error() or b"").decode(errors="replace"), ticket)
        return ticket.out

    def poll_any(self, timeout_ms: int = -1) -> Ticket | None:
        """Process-wide (see :func:`poll_any`): may return a ticket submitted through another model."""
        return poll_any(timeout_ms)

    def embed(self, ids: np.ndarray, lens=None) -> np.ndarray:
        """Synchronous convenience: one input in, its embeddings out.  The caller is blocked for the duration, so a
        C-contiguous int32 ``ids`` is lent to the library instead of copied."""
        lend = isinstance(ids, np.ndarray) and ids.dtype == np.int32 and ids.flags.c_contiguous
        return self.wait(self.submit(ids, lens, borrow_ids=lend))

    def wave_capacity_items(self) -> int:
        """Items of 512 tokens one replica takes per wave of this model: :func:`wave_capacity_items` for bge-base and
        bge-small, 3/4 of it for bge-large (99 on an H100 SXM), whose 1024-wide rows fill the same workspace sooner."""
        return _check(self._lib.b200rt_model_wave_capacity_items(self.handle))

    def debug_cap_rows(self) -> int:
        """Rows of this model one replica's workspace holds, as the engine records them (b200rt_debug_model_cap_rows): 512
        :func:`wave_capacity_items` for bge-base and bge-small, 3/4 of that rounded down to 128 for bge-large."""
        return _check(self._lib.b200rt_debug_model_cap_rows(self.handle))

    def embed_device(self, gpu: int, d_ids: int, d_lens: int, n_items: int, max_len: int, d_out: int, stream: int = 0):
        """Device-resident forward (raw device addresses); asynchronous on ``stream``."""
        _check(self._lib.b200rt_embed_device(self.handle, gpu, d_ids, d_lens, n_items, max_len, d_out, stream or None))

    # ---- debug helpers (tests only)
    def debug_trace(self, ids: np.ndarray, lens, n_launches: int) -> dict:
        """The workspace after the first ``n_launches`` launches of this batch's forward (see :func:`_debug_trace`)."""
        return self._trace(ids, lens, None, n_launches)

    def _trace(self, ids, lens, segs, n_launches: int) -> dict:
        """b200rt_debug_forward_trace_segs (segs None: one segment per item, as b200rt_debug_forward_trace)."""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        n, S = ids.shape
        p = lambda v: _ptr(v) if v is not None else None  # noqa: E731
        lens_a, segs_a = (np.ascontiguousarray(v, dtype=np.int32) if v is not None else None for v in (lens, segs))
        return _debug_trace(lambda *bufs: self._lib.b200rt_debug_forward_trace_segs(self.handle, _ptr(ids), p(lens_a), p(segs_a), n, S,
                                                                                    n_launches, *bufs),
                            n * S, n, self.hidden, self.inter, self.out_dim, n_launches, self.debug_cap_rows())

    def debug_residual(self, ids: np.ndarray, lens, n_layers: int) -> np.ndarray:
        """The residual stream after ``n_layers`` encoder layers (0: the embedding sum), pre-LayerNorm as the forward carries
        it: hi + lo, float32 [n_items, max_len, hidden].  The launches before it are embed and 5 per layer."""
        return _residual(self.debug_trace(ids, lens, 1 + 5 * n_layers), len(ids))

    def profile_forward(self, n_items: int, max_len: int, iters: int = 3) -> dict:
        names = ctypes.create_string_buffer(4096)
        ms = (ctypes.c_float * 64)()
        n = ctypes.c_int32(0)
        _check(self._lib.b200rt_debug_profile_forward(self.handle, n_items, max_len, iters, names, 4096, ms, ctypes.byref(n), 64))
        parts = names.raw.split(b"\0")
        return {parts[i].decode(): float(ms[i]) for i in range(n.value)}


class ClipTextModel(EmbedModel):
    """A loaded CLIP text tower (kind "clip_text"): token ids in, ``[n, proj]`` unit-norm embeddings out -- the in-box
    stand-in for infinity's ``engine.embed(sentences=...)`` on the reference's CLIP model (image_embeddings_infinity.py:298-306).
    ``submit``/``wait``/``embed``/``debug_trace`` are :class:`EmbedModel`'s: same tickets, same scheduler, width ``proj``.
    Token ids come from infinity_emb.clip_tokenizer (``<|startoftext|>`` ... ``<|endoftext|>``, at most ``max_pos``)."""

    def __init__(self, geometry: dict, blob: np.ndarray):
        g = geometry
        self.hidden, self.inter, self.proj = g["hidden"], g["inter"], g["proj"]
        self.out_dim = self.proj
        self.pooling = "eos"
        cfg = ClipTextConfig(g["vocab"], g["hidden"], g["layers"], g["heads"], g["inter"], g["max_pos"], g["proj"], g["eos_id"], g["eps"])
        _load(self, b"clip_text", cfg, blob)


class ClassifierModel(EmbedModel):
    """A loaded BERT sequence classifier / cross-encoder (kind "bert_classifier", HF ``BertForSequenceClassification``):
    token ids in -- single sequences, or ``[CLS] a [SEP] b [SEP]`` pairs whose second segment starts at ``segs[i]`` --
    ``[n, num_labels]`` raw logits out.  TEI serves such a model through ``/rerank`` (``num_labels == 1``: a relevance logit per
    (query, text) pair) and ``/predict``; the sigmoid / softmax is the caller's.  ``submit``/``wait``/``poll_any`` are
    :class:`EmbedModel`'s: same tickets, same scheduler, width ``num_labels``."""

    def __init__(self, geometry: dict, blob: np.ndarray):
        g = geometry
        self.hidden, self.inter, self.num_labels = g["hidden"], g["inter"], g["num_labels"]
        self.out_dim = self.num_labels
        self.pooling = "cls_head"
        _load(self, b"bert_classifier", BertClassifierConfig(_bert_config(g), g["num_labels"]), blob)

    def submit(self, ids: np.ndarray, lens=None, out: np.ndarray | None = None, tag=None, borrow_ids: bool = False, segs=None) -> Ticket:
        """As :meth:`EmbedModel.submit`; ``segs`` [n_items]: where each item's second segment starts (0 <= segs[i] <= lens[i];
        None: one segment)."""
        return self._submit(ids, lens, segs, out, tag, borrow_ids)

    def classify(self, ids: np.ndarray, lens=None, segs=None) -> np.ndarray:
        """Synchronous: ``[n, num_labels]`` raw logits of one batch."""
        lend = isinstance(ids, np.ndarray) and ids.dtype == np.int32 and ids.flags.c_contiguous
        return self.wait(self.submit(ids, lens, borrow_ids=lend, segs=segs))

    def embed_device(self, gpu: int, d_ids: int, d_lens: int, n_items: int, max_len: int, d_out: int, stream: int = 0, d_segs: int = 0):
        """Device-resident forward (raw device addresses; ``d_segs`` 0: one segment); asynchronous on ``stream``."""
        _check(self._lib.b200rt_embed_device_pairs(self.handle, gpu, d_ids, d_lens, d_segs or None, n_items, max_len, d_out, stream or None))

    def debug_trace(self, ids: np.ndarray, lens, n_launches: int, segs=None) -> dict:
        """The workspace after the first ``n_launches`` launches of this batch's forward (see :func:`_debug_trace`); the last
        launch is ``cls_head``, whose logits come back as ``out``."""
        return self._trace(ids, lens, segs, n_launches)


class SparseEmbedModel(EmbedModel):
    """A loaded SPLADE sparse encoder (kind "bert_splade": HF ``BertForMaskedLM`` + sentence-transformers'
    ``SpladePooling(max, relu)``, e.g. naver/splade-v3): token ids in, ``[n, vocab]`` float32 out, ``log(1 + max over the item's
    tokens of relu(MLM logit))`` -- mostly zeros, unnormalised.  TEI serves such a model through ``/embed_sparse``.
    ``submit``/``wait``/``poll_any``/``embed_device`` are :class:`EmbedModel`'s: same tickets, same scheduler, width ``vocab``;
    ``embed_device`` takes ``max_len`` a multiple of 64."""

    def __init__(self, geometry: dict, blob: np.ndarray):
        g = geometry
        self.hidden, self.inter, self.vocab = g["hidden"], g["inter"], g["vocab"]
        self.out_dim = self.vocab
        self.pooling = "splade"
        _load(self, b"bert_splade", _bert_config(g), blob)


class NomicEmbedModel(EmbedModel):
    """A loaded nomic-bert encoder (kind "nomic_bert", HF ``NomicBertModel``: nomic-ai/nomic-embed-text-v1 / -v1.5): rotary
    positions, SwiGLU MLPs, inputs up to ``max_pos`` (at most 8192) tokens.  ``geometry`` is bge-base's plus ``rope_theta``
    (b200rt.weights.NOMIC_EMBED_TEXT_GEOMETRY), the blob b200rt.weights.nomic_blob_layout's.  ``pooling``: "mean" (the
    sentence-transformers pooling nomic-embed-text ships) or "cls"; either way L2-normalised 768-vectors.  ``submit``/``wait``/
    ``embed``/``debug_trace`` are :class:`EmbedModel`'s; items travel in 64-token buckets up to max_pos, and ``embed_device``
    takes ``max_len`` a multiple of 64."""

    def __init__(self, geometry: dict, blob: np.ndarray, pooling: str = "mean"):
        g = geometry
        self.hidden, self.inter, self.max_pos = g["hidden"], g["inter"], g["max_pos"]
        self.out_dim = self.hidden
        self.pooling = pooling
        _load(self, b"nomic_bert", NomicBertConfig(_bert_config(g), g["rope_theta"]), blob, _pool_flags(pooling))


class ImageEmbedModel:
    """A loaded CLIP-style ViT image tower (kind "vit"): ``submit``/``wait`` take preprocessed pixels
    ``[n, 3, image, image]`` float32 and give ``[n, proj]`` unit-norm embeddings -- the in-box stand-in for
    ``engine.image_embed(images=...)`` in the reference's image example (image_embeddings_infinity.py:330-350)."""

    def __init__(self, geometry: dict, blob: np.ndarray):
        g = geometry
        self.image, self.proj = g["image"], g["proj"]
        self.tokens = (g["image"] // g["patch"]) ** 2 + 1
        self.hidden, self.inter = g["hidden"], g["inter"]
        _load(self, b"vit", VitConfig(g["image"], g["patch"], g["hidden"], g["layers"], g["heads"], g["inter"], g["proj"], g["eps"]), blob)

    def submit(self, pixels: np.ndarray, out: np.ndarray | None = None, tag=None) -> Ticket:
        """``pixels`` (C-contiguous float32) and ``out`` stay lent to the library until the ticket completes."""
        if not (isinstance(pixels, np.ndarray) and pixels.dtype == np.float32 and pixels.flags.c_contiguous):
            pixels = np.ascontiguousarray(pixels, dtype=np.float32)
        if pixels.ndim != 4 or pixels.shape[1:] != (3, self.image, self.image):
            raise B200RTError(E_INVALID, f"pixels must be [n, 3, {self.image}, {self.image}], got shape {pixels.shape}")
        n = pixels.shape[0]
        if out is None:
            out = np.empty((n, self.proj), np.float32)
        elif out.dtype != np.float32 or not out.flags.c_contiguous or out.shape != (n, self.proj):
            raise B200RTError(E_INVALID, "out must be a C-contiguous float32 [n_items, proj] array")
        t = ctypes.c_uint64(0)
        with _live_lock:
            _check(self._lib.b200rt_submit_pixels(self.handle, _ptr(pixels), n, _ptr(out), ctypes.byref(t)))
            tk = Ticket(t.value, out, tag, pixels)
            _live[tk.id] = tk
        return tk

    wait = EmbedModel.wait
    poll_any = EmbedModel.poll_any

    def embed(self, pixels: np.ndarray) -> np.ndarray:
        return self.wait(self.submit(pixels))

    def debug_trace(self, pixels: np.ndarray, n_launches: int) -> dict:
        """The workspace after the first ``n_launches`` launches of this batch's forward (see :func:`_debug_trace`)."""
        pixels = np.ascontiguousarray(pixels, dtype=np.float32)
        n = pixels.shape[0]
        return _debug_trace(lambda *bufs: self._lib.b200rt_debug_vit_forward_trace(self.handle, _ptr(pixels), n, n_launches, *bufs),
                            n * self.tokens, n, self.hidden, self.inter, self.proj, n_launches)

    def debug_residual(self, pixels: np.ndarray, n_layers: int) -> np.ndarray:
        """The residual stream after ``n_layers`` encoder layers (0: the pre_layrnorm output): hi + lo, float32
        [n_items, tokens, hidden].  The launches before it are im2col, gemm_patch, vit_embed and 5 per layer."""
        return _residual(self.debug_trace(pixels, 3 + 5 * n_layers), len(pixels))


_TRACE_NAMES_CAP = 8192


def _debug_trace(call, M: int, n_items: int, H: int, I: int, out_dim: int, n_launches: int, cap_rows: int | None = None) -> dict:
    """One b200rt_debug_*forward_trace call (include/b200rt_debug.h).  Returns the workspace, each buffer for
    ``rows = min(M + 256, cap_rows)`` rows (cap_rows: the model's workspace rows as the engine reports them; by default the
    runtime's):
    yhi, ylo, ctx float16 [rows, H]; qkv float16 [rows, 3H]; ffn float16 [rows, I];
    pstats0, pstats1 float32 [rows, H / 128, 2]; ``out`` [n_items, out_dim] once the pool launch has run (else None);
    ``names`` of the launches run, ``n_total`` launches in the whole forward, ``M`` and ``rows``."""
    rows = min(M + 256, cap_rows if cap_rows is not None else wave_capacity_items() * 512)
    P = H // 128
    bufs = dict(yhi=np.empty((rows, H), np.float16), ylo=np.empty((rows, H), np.float16),
                pstats0=np.empty((rows, P, 2), np.float32), pstats1=np.empty((rows, P, 2), np.float32),
                qkv=np.empty((rows, 3 * H), np.float16), ctx=np.empty((rows, H), np.float16), ffn=np.empty((rows, I), np.float16))
    out = np.empty((n_items, out_dim), np.float32)
    names = ctypes.create_string_buffer(_TRACE_NAMES_CAP)
    total = ctypes.c_int32(0)
    order = ("yhi", "ylo", "pstats0", "pstats1", "qkv", "ctx", "ffn")
    _check(call(*(_ptr(bufs[k]) for k in order), _ptr(out), names, _TRACE_NAMES_CAP, ctypes.byref(total)))
    bufs.update(out=out if n_launches == total.value else None, names=[s.decode() for s in names.raw.split(b"\0")[:n_launches]],
                n_total=total.value, M=M, rows=rows)
    return bufs


def _residual(trace: dict, n_items: int) -> np.ndarray:
    """hi + lo of a trace's M rows, [n_items, M / n_items, hidden] float32 (the sum the row kernels form)."""
    M = trace["M"]
    return (trace["yhi"][:M].astype(np.float32) + trace["ylo"][:M].astype(np.float32)).reshape(n_items, M // n_items, -1)


def device_sync(gpu: int = 0):
    _check(load_library().b200rt_device_sync(gpu))


def debug_gemm(epi: int, a16: np.ndarray, w16: np.ndarray, bias: np.ndarray, resid=None, iters: int = 1, ln_stats=None,
               ln_gamma=None, ln_beta=None, eps: float = 1e-12, want_stats: bool = False, sms: int = 0, want_ctas: bool = False,
               ln512: bool = False):
    """a16 [M,K], w16 [N,K] float16; returns (out, ms) -- or (out, ms, stats_out [M, N/128, 2]) with ``want_stats`` (epi 2),
    and with ``want_ctas`` the number of CTAs launched appended.
    ``ln_stats`` [M, parts, 2] (sum, M2) partials switch the LayerNorm epilogues on (see include/b200rt_debug.h).
    ``sms``: the most CTAs of the persistent launch (0 = every SM), rounded down to whole 2-CTA clusters, at least one.
    ``ln512``: also accept a 512-wide LayerNorm (the CLIP text tower's 4-partial epilogues; b200rt_debug_gemm_ex)."""
    a16 = np.ascontiguousarray(a16, dtype=np.float16)
    w16 = np.ascontiguousarray(w16, dtype=np.float16)
    bias = np.ascontiguousarray(bias, dtype=np.float32)
    M, K = a16.shape
    N = w16.shape[0]
    out = np.empty((M, N), np.float32 if epi == 2 else np.float16)
    c32 = lambda v: np.ascontiguousarray(v, dtype=np.float32) if v is not None else None  # noqa: E731
    r, st, lg, lb = c32(resid), c32(ln_stats), c32(ln_gamma), c32(ln_beta)
    so = np.zeros((M, N // 128, 2), np.float32) if want_stats else None
    p = lambda v: _ptr(v) if v is not None else None  # noqa: E731
    ms = ctypes.c_float(0)
    ctas = ctypes.c_int(0)
    _check(load_library().b200rt_debug_gemm_ex(epi, _ptr(a16), _ptr(w16), _ptr(bias), p(r), _ptr(out), M, N, K, iters, ctypes.byref(ms),
                                               p(st), p(lg), p(lb), eps, p(so), sms, ctypes.byref(ctas), DEBUG_GEMM_LN512 if ln512 else 0))
    res = (out, ms.value, so) if want_stats else (out, ms.value)
    return res + (ctas.value,) if want_ctas else res


DEBUG_ATTN_CAUSAL = 1
DEBUG_GEMM_LN512 = 1


def debug_attention(qkv16: np.ndarray, lens: np.ndarray, B: int, S: int, iters: int = 1, sms: int = 0, head_dim: int = 64,
                    heads: int = 12, causal: bool = False):
    """qkv16 [B*S, 3H] float16 with H = heads head_dim ((64, 12): bge-base, (32, 12): bge-small, (64, 16): bge-large;
    causal (64, 8): the CLIP text tower); returns (ctx [B*S, H], ms)."""
    H = heads * head_dim
    qkv16 = np.ascontiguousarray(qkv16, dtype=np.float16)
    if qkv16.size != B * S * 3 * H:
        raise B200RTError(E_INVALID, f"qkv must be [{B * S}, {3 * H}] for {heads} heads of {head_dim}, got shape {qkv16.shape}")
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    ctx = np.empty((B * S, H), np.float16)
    ms = ctypes.c_float(0)
    _check(load_library().b200rt_debug_attention_ex(_ptr(qkv16), _ptr(lens), _ptr(ctx), B, S, iters, ctypes.byref(ms), sms, head_dim, heads,
                                                 DEBUG_ATTN_CAUSAL if causal else 0))
    return ctx, ms.value


# Row kernels behind host buffers (include/b200rt_debug.h).  hi / lo are float16 arrays [rows, W]; stats [rows, W / 128, 2];
# W = 768, or ``hidden`` (768, 384 or 1024) where a wrapper takes it.
def _f32(v):
    return np.ascontiguousarray(v, dtype=np.float32)


def _f16(v):
    return np.ascontiguousarray(v, dtype=np.float16)


def debug_embed(ids: np.ndarray, word: np.ndarray, pos: np.ndarray, type0: np.ndarray, S: int, hidden: int = 768):
    """ids [n_tokens] (token t sits at position t % S), word [vocab, hidden], pos [S, hidden]; returns (hi, lo, stats)."""
    ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
    word, pos, type0 = _f32(word), _f32(pos), _f32(type0)
    if word.shape[1] != hidden or pos.shape[1] != hidden or type0.size != hidden:
        raise B200RTError(E_INVALID, f"embedding tables must be {hidden} wide")
    n = ids.size
    hi, lo = np.empty((n, hidden), np.float16), np.empty((n, hidden), np.float16)
    st = np.empty((n, hidden // 128, 2), np.float32)
    _check(load_library().b200rt_debug_embed(_ptr(ids), _ptr(word), _ptr(pos), _ptr(type0), n, S, word.shape[0], _ptr(hi), _ptr(lo), _ptr(st),
                                             hidden))
    return hi, lo, st


def debug_embed_segs(ids: np.ndarray, segs, word: np.ndarray, pos: np.ndarray, type2: np.ndarray, S: int, hidden: int = 768):
    """ids [n_items * S] (token t sits at position t % S of item t // S), segs [n_items] (passed as given; the kernel clamps each
    to [0, S]), type2 [2, hidden]: token t takes type row 1 when t % S >= segs[t // S]; returns (hi, lo, stats)."""
    ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
    segs = np.ascontiguousarray(segs, dtype=np.int32).reshape(-1)
    word, pos, type2 = _f32(word), _f32(pos), _f32(type2)
    if word.shape[1] != hidden or pos.shape[1] != hidden or type2.shape != (2, hidden):
        raise B200RTError(E_INVALID, f"embedding tables must be {hidden} wide and type2 [2, {hidden}]")
    n = ids.size
    if n % S or segs.size != n // S:
        raise B200RTError(E_INVALID, f"ids must hold whole items of {S} tokens and segs one entry per item")
    hi, lo = np.empty((n, hidden), np.float16), np.empty((n, hidden), np.float16)
    st = np.empty((n, hidden // 128, 2), np.float32)
    _check(load_library().b200rt_debug_embed_segs(_ptr(ids), _ptr(segs), _ptr(word), _ptr(pos), _ptr(type2), n, S, word.shape[0], _ptr(hi),
                                                  _ptr(lo), _ptr(st), hidden))
    return hi, lo, st


def debug_cls_head(hi: np.ndarray, lo: np.ndarray, gamma, beta, pool_w, pool_b, cls_w, cls_b, S: int, eps: float, hidden: int = 768,
                   ctas: int = 0):
    """hi, lo [n_items * S, hidden], pool_w [hidden, hidden], cls_w [L, hidden]: the raw logits
    cls_w . tanh(pool_w . LayerNorm(row i * S) + pool_b) + cls_b, [n_items, L].  ``ctas``: the most blocks (0 = one per item)."""
    hi, lo, gamma, beta = _f16(hi), _f16(lo), _f32(gamma), _f32(beta)
    pool_w, pool_b, cls_w, cls_b = _f32(pool_w), _f32(pool_b), _f32(cls_w), _f32(cls_b)
    L = cls_w.shape[0]
    if hi.shape[1] != hidden or pool_w.shape != (hidden, hidden) or cls_w.shape[1] != hidden or cls_b.size < L:
        raise B200RTError(E_INVALID, f"rows and head weights must be {hidden} wide")
    n = hi.shape[0] // S
    out = np.empty((n, max(L, 1)), np.float32)
    _check(load_library().b200rt_debug_cls_head(_ptr(hi), _ptr(lo), _ptr(gamma), _ptr(beta), _ptr(pool_w), _ptr(pool_b), _ptr(cls_w),
                                                _ptr(cls_b), n, S, L, eps, _ptr(out), hidden, ctas))
    return out


def debug_vit_embed(patch_out: np.ndarray, cls: np.ndarray, pos: np.ndarray, gamma: np.ndarray, beta: np.ndarray, T: int, eps: float):
    """patch_out [rows, 768] float16 (row t is token t % T); returns (hi, lo, stats)."""
    patch_out, cls, pos, gamma, beta = _f16(patch_out), _f32(cls), _f32(pos), _f32(gamma), _f32(beta)
    n = patch_out.shape[0]
    hi, lo = np.empty((n, 768), np.float16), np.empty((n, 768), np.float16)
    st = np.empty((n, 6, 2), np.float32)
    _check(load_library().b200rt_debug_vit_embed(_ptr(patch_out), _ptr(cls), _ptr(pos), _ptr(gamma), _ptr(beta), n, T, eps,
                                                 _ptr(hi), _ptr(lo), _ptr(st)))
    return hi, lo, st


def debug_pool_normalize(hi: np.ndarray, lo: np.ndarray, gamma: np.ndarray, beta: np.ndarray, S: int, eps: float, hidden: int = 768):
    """hi, lo [n_items * S, hidden]: the LayerNorm'd, L2-normalised row i * S of every item, [n_items, hidden]."""
    hi, lo, gamma, beta = _f16(hi), _f16(lo), _f32(gamma), _f32(beta)
    if hi.shape[1] != hidden or lo.shape[1] != hidden or gamma.size != hidden or beta.size != hidden:
        raise B200RTError(E_INVALID, f"rows and LayerNorm parameters must be {hidden} wide")
    n = hi.shape[0] // S
    out = np.empty((n, hidden), np.float32)
    _check(load_library().b200rt_debug_pool_normalize(_ptr(hi), _ptr(lo), _ptr(gamma), _ptr(beta), n, S, eps, _ptr(out), hidden))
    return out


def debug_mean_pool_normalize(hi: np.ndarray, lo: np.ndarray, gamma: np.ndarray, beta: np.ndarray, lens, S: int, eps: float,
                              hidden: int = 768):
    """hi, lo [n_items * S, hidden], lens [n_items] (passed to the device as given; the kernel clamps each to [1, S]): the
    L2-normalised mean of the LayerNorm'd rows i * S + r, r < lens[i], of every item, [n_items, hidden]."""
    hi, lo, gamma, beta = _f16(hi), _f16(lo), _f32(gamma), _f32(beta)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    if hi.shape[1] != hidden or lo.shape[1] != hidden or gamma.size != hidden or beta.size != hidden:
        raise B200RTError(E_INVALID, f"rows and LayerNorm parameters must be {hidden} wide")
    n = hi.shape[0] // S
    if lens.shape != (n,):
        raise B200RTError(E_INVALID, f"lens must have shape ({n},), got {lens.shape}")
    out = np.empty((n, hidden), np.float32)
    _check(load_library().b200rt_debug_mean_pool_normalize(_ptr(hi), _ptr(lo), _ptr(gamma), _ptr(beta), _ptr(lens), n, S, eps, _ptr(out),
                                                           hidden))
    return out


def debug_vit_pool(hi: np.ndarray, lo: np.ndarray, gamma: np.ndarray, beta: np.ndarray, proj: np.ndarray, T: int, eps: float):
    """hi, lo [n_items * T, 768], proj [P, 768]: normalise(proj . LayerNorm(row i * T)), [n_items, P]."""
    hi, lo, gamma, beta, proj = _f16(hi), _f16(lo), _f32(gamma), _f32(beta), _f32(proj)
    n, P = hi.shape[0] // T, proj.shape[0]
    out = np.empty((n, max(P, 1)), np.float32)
    _check(load_library().b200rt_debug_vit_pool(_ptr(hi), _ptr(lo), _ptr(gamma), _ptr(beta), _ptr(proj), n, T, P, eps, _ptr(out)))
    return out


def debug_clip_text_pool(hi: np.ndarray, lo: np.ndarray, ids: np.ndarray, lens, gamma: np.ndarray, beta: np.ndarray, proj: np.ndarray,
                         S: int, eps: float, eos_id: int):
    """hi, lo [n_items * S, 512], ids [n_items, S], lens [n_items] (clamped to [1, S] on the device), proj [P, 512]:
    normalise(proj . LayerNorm(row i * S + p_i)) with p_i the item's pooled position, [n_items, P]."""
    hi, lo, gamma, beta, proj = _f16(hi), _f16(lo), _f32(gamma), _f32(beta), _f32(proj)
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    n, P = hi.shape[0] // S, proj.shape[0]
    if ids.size != n * S or lens.shape != (n,):
        raise B200RTError(E_INVALID, f"ids must be [{n}, {S}] and lens [{n}]")
    out = np.empty((n, max(P, 1)), np.float32)
    _check(load_library().b200rt_debug_clip_text_pool(_ptr(hi), _ptr(lo), _ptr(ids), _ptr(lens), _ptr(gamma), _ptr(beta), _ptr(proj), n, S, P,
                                                      eps, eos_id, _ptr(out)))
    return out


def debug_fold_ln(w: np.ndarray, gamma=None, beta=None, bias=None):
    """w [N, K] float32; returns (w_out float16 [N, K], cvec [N] or None when gamma is None)."""
    w = _f32(w)
    N, K = w.shape
    p = lambda v: _ptr(v) if v is not None else None  # noqa: E731
    g, b, bs = (_f32(v) if v is not None else None for v in (gamma, beta, bias))
    w_out = np.empty((N, K), np.float16)
    cvec = np.empty(N, np.float32) if gamma is not None else None
    _check(load_library().b200rt_debug_fold_ln(_ptr(w), p(g), p(b), p(bs), N, K, _ptr(w_out), p(cvec)))
    return w_out, cvec


def debug_gemm_splade(a16: np.ndarray, w16: np.ndarray, c, stats, lens, S: int, N: int, eps: float, sms: int = 0, iters: int = 1,
                      want_ctas: bool = False):
    """The SPLADE decoder GEMM (b200rt_debug_gemm_splade): a16 [B S, K], w16 [vocab, K] float16, c [N], stats [B S, K / 128, 2],
    lens [B]; returns (uint32 maxima [B, N] -- the fp32 bits of max(0, max over item i's valid rows) --, ms per launch), and
    with ``want_ctas`` the number of CTAs launched appended."""
    a16 = np.ascontiguousarray(a16, dtype=np.float16)
    w16 = np.ascontiguousarray(w16, dtype=np.float16)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    c, stats = _f32(c), _f32(stats)
    B, K, vocab = len(lens), a16.shape[1], w16.shape[0]
    out = np.empty((B, N), np.uint32)
    ms = ctypes.c_float(0)
    ctas = ctypes.c_int(0)
    _check(load_library().b200rt_debug_gemm_splade(_ptr(a16), _ptr(w16), _ptr(c), _ptr(stats), _ptr(lens), B, S, N, K, vocab,
                                                   eps, sms, iters, ctypes.byref(ms), _ptr(out), ctypes.byref(ctas)))
    return (out, ms.value, ctas.value) if want_ctas else (out, ms.value)


def debug_mlm_ln_stats(u16: np.ndarray, n_max: int = 0):
    """(stats [rows, W / 128, 2] of the fp16 rows u16 [rows, W], the n_max-word max buffer as the launch leaves it)."""
    u16 = np.ascontiguousarray(u16, dtype=np.float16)
    rows, W = u16.shape
    st = np.empty((rows, W // 128, 2), np.float32)
    vmax = np.empty(max(n_max, 1), np.uint32)
    _check(load_library().b200rt_debug_mlm_ln_stats(_ptr(u16), rows, W, n_max, _ptr(vmax), _ptr(st)))
    return st, vmax[:n_max]


def debug_splade_finalize(vmax: np.ndarray, vocab: int) -> np.ndarray:
    """log1p of the fp32 bits of uint32 vmax [n, vpad], first ``vocab`` columns: float32 [n, vocab]."""
    vmax = np.ascontiguousarray(vmax, dtype=np.uint32)
    n, vpad = vmax.shape
    out = np.empty((n, vocab), np.float32)
    _check(load_library().b200rt_debug_splade_finalize(_ptr(vmax), n, vpad, vocab, _ptr(out)))
    return out


def debug_gemm_rope(a16: np.ndarray, w16: np.ndarray, c, stats, table: np.ndarray, S: int, rot_cols: int, eps: float, sms: int = 0,
                    want_ctas: bool = False):
    """nomic-bert's QKV epilogue (b200rt_debug_gemm_rope): a16 [M, 768], w16 [N, 768] float16, c [N], stats [M, 6, 2] or None,
    table float32 [n_pos, 32, 2] (cos, sin); returns out float16 [M, N], or (out, CTAs launched) with ``want_ctas``."""
    a16 = np.ascontiguousarray(a16, dtype=np.float16)
    w16 = np.ascontiguousarray(w16, dtype=np.float16)
    M, N = a16.shape[0], w16.shape[0]
    c, table = _f32(c), _f32(table)
    st = _f32(stats) if stats is not None else None
    out = np.empty((M, N), np.float16)
    ctas = ctypes.c_int(0)
    _check(load_library().b200rt_debug_gemm_rope(_ptr(a16), _ptr(w16), _ptr(c), _ptr(st) if st is not None else None, _ptr(table),
                                                 table.shape[0], M, N, S, rot_cols, eps, sms, _ptr(out), ctypes.byref(ctas)))
    return (out, ctas.value) if want_ctas else out


def debug_gemm_swiglu(a16: np.ndarray, w16: np.ndarray, c, stats, eps: float, sms: int = 0, want_ctas: bool = False):
    """nomic-bert's FFN1 epilogue (b200rt_debug_gemm_swiglu): w16 [N, 768] with gate / up rows interleaved in groups of 8, c [N];
    returns out float16 [M, N / 2] = silu(g) u, or (out, CTAs launched) with ``want_ctas``."""
    a16 = np.ascontiguousarray(a16, dtype=np.float16)
    w16 = np.ascontiguousarray(w16, dtype=np.float16)
    M, N = a16.shape[0], w16.shape[0]
    c = _f32(c)
    st = _f32(stats) if stats is not None else None
    out = np.empty((M, N // 2), np.float16)
    ctas = ctypes.c_int(0)
    _check(load_library().b200rt_debug_gemm_swiglu(_ptr(a16), _ptr(w16), _ptr(c), _ptr(st) if st is not None else None, M, N, eps, sms,
                                                   _ptr(out), ctypes.byref(ctas)))
    return (out, ctas.value) if want_ctas else out


def debug_attention_stream(qkv16: np.ndarray, lens, B: int, S: int, sms: int = 0, iters: int = 0):
    """The streaming K/V attention (b200rt_debug_attention_stream): qkv16 [B*S, 2304] float16; returns (ctx [B*S, 768] float16,
    mean ms of ``iters`` further launches, 0 when iters == 0)."""
    qkv16 = np.ascontiguousarray(qkv16, dtype=np.float16)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    ctx = np.empty((B * S, 768), np.float16)
    ms = ctypes.c_float(0)
    _check(load_library().b200rt_debug_attention_stream(_ptr(qkv16), _ptr(lens), B, S, _ptr(ctx), sms, iters, ctypes.byref(ms)))
    return ctx, ms.value
