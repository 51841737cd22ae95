"""``text-embeddings-router`` stand-in.  Flags as the reference passes them
(``text_embeddings_inference.py:29-34``, ``amazon_embeddings.py:283-294``, ``wikipedia/main.py:42-53``); it binds
127.0.0.1:PORT only after the weights are resident on every replica, so the reference's TCP readiness poll
(``text_embeddings_inference.py:41-51``) means what it meant with TEI; exits non-zero when the engine cannot
start (the poll loop then raises "launcher exited unexpectedly")."""
from __future__ import annotations

import argparse
import json
import os
import sys
import threading
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer

GEOMETRY = dict(vocab=30522, hidden=768, layers=12, heads=12, inter=3072, max_pos=512, type_vocab=2, eps=1e-12)
BGE_SMALL_ID = "BAAI/bge-small-en-v1.5"
BGE_LARGE_ID = "BAAI/bge-large-en-v1.5"


MINILM_L6_ID = "sentence-transformers/all-MiniLM-L6-v2"
POOLING_BY_MODEL_ID = {MINILM_L6_ID: "mean"}  # models whose sentence-transformers config pools other than by [CLS]
POOLINGS = ("cls", "mean")  # TEI also knows splade and last-token; this runtime does not


def geometry_for_model_id(model_id: str) -> dict:
    """Geometry of the offline seeded fallback and of a raw --weights blob (which carries no shapes): bge-small's for
    BAAI/bge-small-en-v1.5, bge-large's for BAAI/bge-large-en-v1.5, MiniLM-L6's (bge-small's with 6 layers) for
    sentence-transformers/all-MiniLM-L6-v2, bge-base's for BAAI/bge-base-en-v1.5 and for any id this table does not know.
    A hub snapshot takes its geometry from its own config.json instead."""
    from b200rt.weights import BGE_BASE_GEOMETRY, BGE_LARGE_GEOMETRY, BGE_SMALL_GEOMETRY, MINILM_L6_GEOMETRY

    known = {"BAAI/bge-base-en-v1.5": BGE_BASE_GEOMETRY, BGE_SMALL_ID: BGE_SMALL_GEOMETRY, BGE_LARGE_ID: BGE_LARGE_GEOMETRY,
             MINILM_L6_ID: MINILM_L6_GEOMETRY}
    return dict(known.get(model_id, BGE_BASE_GEOMETRY))


def resolve_pooling(flag: str | None, snapshot_dir: str | None, model_id: str) -> str:
    """The pooling to serve, resolved as TEI resolves it: --pooling when given; else the Pooling module of the snapshot's
    sentence-transformers config (modules.json -> 1_Pooling/config.json); else the model-id table; else cls.  Raises
    ValueError for a --pooling other than cls / mean and for a snapshot that declares a pooling other than those two."""
    from b200rt.weights import pooling_from_dir

    if flag is not None:
        if flag not in POOLINGS:
            raise ValueError(f"--pooling {flag!r} is not supported (supported: {', '.join(POOLINGS)})")
        return flag
    if snapshot_dir:
        declared = pooling_from_dir(snapshot_dir)
        if declared is not None:
            return declared
    return POOLING_BY_MODEL_ID.get(model_id, "cls")


def parse_args(argv):
    ap = argparse.ArgumentParser(prog="text-embeddings-router", allow_abbrev=False)
    ap.add_argument("--model-id", default="BAAI/bge-base-en-v1.5")
    ap.add_argument("--port", type=int, default=int(os.environ.get("PORT", "3000")))
    ap.add_argument("--hostname", default="127.0.0.1")
    ap.add_argument("--max-client-batch-size", type=int, default=32)
    ap.add_argument("--max-batch-tokens", type=int, default=16384)
    ap.add_argument("--max-concurrent-requests", type=int, default=512)
    ap.add_argument("--huggingface-hub-cache", default=None)
    ap.add_argument("--revision", default=None)
    ap.add_argument("--dtype", default="float16")
    ap.add_argument("--pooling", default=None, help="cls or mean; default: the snapshot's sentence-transformers Pooling config, else cls")
    ap.add_argument("--auto-truncate", action="store_true")
    ap.add_argument("--tokenizer-vocab", default=os.environ.get("B200RT_VOCAB"))
    ap.add_argument("--weights", default=os.environ.get("B200RT_WEIGHTS"), help="flat fp32 blob (DESIGN.md §3), a .safetensors checkpoint or an HF snapshot directory; default: the hub cache, else seeded random init")
    ap.add_argument("--gpus", type=int, default=int(os.environ.get("B200RT_GPUS", "0")), help="0 = all visible")
    args, unknown = ap.parse_known_args(argv)
    if unknown:
        print(f"[text-embeddings-router/b200] ignoring unsupported flags: {unknown}", file=sys.stderr)
    return args


def random_blob(seed=0, geometry=None):
    """Seeded weights of `geometry` (default BGE-base; the one definition lives in b200rt.weights)."""
    from b200rt.weights import random_blob as rb

    return rb(geometry or GEOMETRY, seed)


def weights_dir(args) -> str | None:
    """The directory the weights come from (an HF snapshot directory or the one holding a .safetensors checkpoint), which
    is where a sentence-transformers model keeps modules.json; None for a flat blob or the seeded fallback."""
    from b200rt import weights as W

    if args.weights:
        if os.path.isdir(args.weights):
            return args.weights
        return os.path.dirname(os.path.abspath(args.weights)) if args.weights.endswith(".safetensors") else None
    cache = args.huggingface_hub_cache or os.environ.get("HUGGINGFACE_HUB_CACHE") or os.environ.get("HF_HUB_CACHE")
    return W.resolve_hub_snapshot(cache, args.model_id) if cache else None


def load_weights(args):
    """Weights for --model-id: an explicit --weights file (flat fp32 blob, or a .safetensors checkpoint), else the HF
    hub snapshot under --huggingface-hub-cache (what the reference's `download_model` leaves there:
    text_embeddings_inference.py:54-56), else seeded random init with a loud notice (no network in this box)."""
    import numpy as np
    from b200rt import weights as W

    if args.weights:
        if args.weights.endswith(".safetensors"):
            return W.load_safetensors(args.weights) + (f"safetensors {args.weights}",)
        if os.path.isdir(args.weights):
            return W.load_hf_dir(args.weights) + (f"HF directory {args.weights}",)
        return geometry_for_model_id(args.model_id), np.fromfile(args.weights, np.float32), f"flat blob {args.weights}"
    cache = args.huggingface_hub_cache or os.environ.get("HUGGINGFACE_HUB_CACHE") or os.environ.get("HF_HUB_CACHE")
    if cache:
        snap = W.resolve_hub_snapshot(cache, args.model_id)
        if snap:
            return W.load_hf_dir(snap) + (f"hub snapshot {snap}",)
    g = geometry_for_model_id(args.model_id)
    return g, random_blob(geometry=g), None


class Engine:
    def __init__(self, args):
        import numpy as np
        import b200rt
        from .tokenizer import WordPiece, load_vocab

        self.np = np
        self.args = args
        self.pooling = resolve_pooling(args.pooling, weights_dir(args), args.model_id)
        self.tok = WordPiece(load_vocab(args.tokenizer_vocab) if args.tokenizer_vocab else None)
        if self.tok.synthetic:
            print("[text-embeddings-router/b200] no BERT vocabulary available: SYNTHETIC WordPiece vocabulary, auto-truncate on "
                  "(string embeddings are not comparable with the real model's)", file=sys.stderr)
            args.auto_truncate = True
        n_gpus = args.gpus
        if n_gpus <= 0:
            import torch

            n_gpus = max(1, torch.cuda.device_count())
        b200rt.init(n_gpus)
        geometry, blob, source = load_weights(args)
        if source is None:
            print(f"[text-embeddings-router/b200] no weights for {args.model_id!r} offline: seeded random init", file=sys.stderr)
        else:
            print(f"[text-embeddings-router/b200] weights: {source}", file=sys.stderr)
        print(f"[text-embeddings-router/b200] pooling: {self.pooling}", file=sys.stderr)
        self.geometry = geometry
        self.model = b200rt.EmbedModel(geometry, blob, pooling=self.pooling)
        self.n_gpus = n_gpus

    def embed(self, inputs):
        np = self.np
        rows = [self.tok.encode(t, self.geometry["max_pos"], self.args.auto_truncate) for t in inputs]
        lens = np.array([len(r) for r in rows], np.int32)
        ids = np.zeros((len(rows), int(lens.max())), np.int32)
        for i, r in enumerate(rows):
            ids[i, : len(r)] = r
        return self.model.embed(ids, lens)


def make_handler(engine: Engine):
    class Handler(BaseHTTPRequestHandler):
        protocol_version = "HTTP/1.1"

        def log_message(self, *a):  # quiet
            pass

        def _send(self, code, obj):
            body = json.dumps(obj).encode()
            self.send_response(code)
            self.send_header("Content-Type", "application/json")
            self.send_header("Content-Length", str(len(body)))
            self.end_headers()
            self.wfile.write(body)

        def do_GET(self):
            if self.path == "/health":
                self._send(200, {})
            elif self.path == "/info":
                self._send(200, {"model_id": engine.args.model_id, "model_dtype": "float16", "max_client_batch_size": engine.args.max_client_batch_size,
                                 "max_input_length": GEOMETRY["max_pos"], "backend": f"b200rt x{engine.n_gpus}", "pooling": engine.pooling})
            else:
                self._send(404, {"error": "not found", "error_type": "NotFound"})

        def do_POST(self):
            if self.path not in ("/embed", "/"):
                return self._send(404, {"error": "not found", "error_type": "NotFound"})
            try:
                req = json.loads(self.rfile.read(int(self.headers.get("Content-Length", "0"))))
                inputs = req["inputs"]
                if isinstance(inputs, str):
                    inputs = [inputs]
                if not isinstance(inputs, list) or not inputs or not all(isinstance(t, str) for t in inputs):
                    raise TypeError("`inputs` must be a string or a non-empty list of strings")
            except Exception as e:  # noqa: BLE001
                return self._send(422, {"error": f"Failed to deserialize the JSON body: {e}", "error_type": "Validation"})
            if len(inputs) > engine.args.max_client_batch_size:
                return self._send(413, {"error": f"batch size {len(inputs)} > maximum allowed batch size {engine.args.max_client_batch_size}",
                                        "error_type": "Validation"})
            try:
                vecs = engine.embed(inputs)
            except ValueError as e:
                return self._send(413, {"error": str(e), "error_type": "Validation"})
            except Exception as e:  # noqa: BLE001
                return self._send(500, {"error": str(e), "error_type": "Backend"})
            self._send(200, vecs.tolist())

    return Handler


def main(argv=None):
    args = parse_args(sys.argv[1:] if argv is None else argv)
    try:
        engine = Engine(args)
    except Exception as e:  # noqa: BLE001  -- no CPU fallback: the launcher must see the exit
        print(f"[text-embeddings-router/b200] cannot start: {e}", file=sys.stderr)
        return 1
    srv = ThreadingHTTPServer((args.hostname, args.port), make_handler(engine))
    srv.daemon_threads = True
    print(f"[text-embeddings-router/b200] ready on {args.hostname}:{args.port} ({engine.n_gpus} GPU replicas)", file=sys.stderr)
    import signal

    def stop(*_):
        threading.Thread(target=srv.shutdown, daemon=True).start()

    signal.signal(signal.SIGTERM, stop)
    signal.signal(signal.SIGINT, stop)
    srv.serve_forever()
    import b200rt

    b200rt.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
