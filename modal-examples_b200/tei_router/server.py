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
# long-context nomic-bert encoders (kind "nomic_bert", inputs up to 8192 tokens); their sentence-transformers config pools by mean
NOMIC_MODEL_IDS = ("nomic-ai/nomic-embed-text-v1.5", "nomic-ai/nomic-embed-text-v1")
POOLING_BY_MODEL_ID = {MINILM_L6_ID: "mean", **{i: "mean" for i in NOMIC_MODEL_IDS}}  # models whose sentence-transformers config pools other than by [CLS]
POOLINGS = ("cls", "mean")  # TEI also knows splade and last-token; this runtime does not
# SPLADE encoders served offline on seeded weights (bge-base's geometry) when no masked-LM snapshot is at hand; a snapshot
# whose config names BertForMaskedLM, or whose weights carry cls.predictions.transform, serves --pooling splade under any id
SPLADE_MODEL_IDS = ("naver/splade-cocondenser-ensembledistil", "naver/splade-v3")
MS_MARCO_L6_ID = "cross-encoder/ms-marco-MiniLM-L-6-v2"
MS_MARCO_L12_ID = "cross-encoder/ms-marco-MiniLM-L-12-v2"


def geometry_for_model_id(model_id: str) -> dict:
    """Geometry of the offline seeded fallback and of a raw --weights blob (which carries no shapes): bge-small's for
    BAAI/bge-small-en-v1.5, bge-large's for BAAI/bge-large-en-v1.5, MiniLM-L6's (bge-small's with 6 layers) for
    sentence-transformers/all-MiniLM-L6-v2, nomic-embed-text's (rotary, 8192 positions) for the NOMIC_MODEL_IDS, bge-base's for
    BAAI/bge-base-en-v1.5 and for any id this table does not know.  A hub snapshot takes its geometry from its own config.json
    instead."""
    from b200rt.weights import (BGE_BASE_GEOMETRY, BGE_LARGE_GEOMETRY, BGE_SMALL_GEOMETRY, MINILM_L6_GEOMETRY, MS_MARCO_MINILM_L6_GEOMETRY,
                                NOMIC_EMBED_TEXT_GEOMETRY)

    known = {"BAAI/bge-base-en-v1.5": BGE_BASE_GEOMETRY, BGE_SMALL_ID: BGE_SMALL_GEOMETRY, BGE_LARGE_ID: BGE_LARGE_GEOMETRY,
             MINILM_L6_ID: MINILM_L6_GEOMETRY, MS_MARCO_L6_ID: MS_MARCO_MINILM_L6_GEOMETRY,
             MS_MARCO_L12_ID: dict(MS_MARCO_MINILM_L6_GEOMETRY, layers=12), **{i: NOMIC_EMBED_TEXT_GEOMETRY for i in NOMIC_MODEL_IDS}}
    return dict(known.get(model_id, BGE_BASE_GEOMETRY))


# --------------------------------------------------------------------------- classifier scoring (host side, as TEI does it)

def _sigmoid(x):
    import numpy as np

    x = np.asarray(x, np.float64)
    return np.where(x >= 0, 1.0 / (1.0 + np.exp(-np.abs(x))), np.exp(-np.abs(x)) / (1.0 + np.exp(-np.abs(x))))


def label_scores(logits, raw_scores: bool):
    """Per-item label scores from ``[n, L]`` raw logits: the logits themselves (raw_scores), else a sigmoid when L == 1 and a
    softmax over the labels otherwise."""
    import numpy as np

    z = np.asarray(logits, np.float64)
    if raw_scores:
        return z
    if z.shape[1] == 1:
        return _sigmoid(z)
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def rerank_response(logits, texts, raw_scores: bool, return_text: bool) -> list:
    """``[{"index", "score"[, "text"]}]`` sorted by score, highest first (ties keep the input order), from ``[n, 1]`` logits."""
    scores = label_scores(logits, raw_scores)[:, 0]
    order = sorted(range(len(scores)), key=lambda i: -scores[i])
    out = []
    for i in order:
        r = {"index": i, "score": float(scores[i])}
        if return_text:
            r["text"] = texts[i]
        out.append(r)
    return out


def predict_response(logits_row, id2label: dict, raw_scores: bool) -> list:
    """``[{"label", "score"}]`` of one input, sorted by score, highest first."""
    scores = label_scores(logits_row[None, :], raw_scores)[0]
    order = sorted(range(len(scores)), key=lambda j: -scores[j])
    return [{"label": id2label.get(j, f"LABEL_{j}"), "score": float(scores[j])} for j in order]


def parse_predict_inputs(inputs):
    """TEI's /predict ``inputs``: a string, a ``[text, text]`` pair, or a list of those.  Returns (list of str or (str, str),
    whether it was a batch)."""
    def seq(x):
        if isinstance(x, str):
            return x
        if isinstance(x, list) and len(x) == 2 and all(isinstance(t, str) for t in x):
            return (x[0], x[1])
        raise TypeError("each input must be a string or a [string, string] pair")

    if isinstance(inputs, str):
        return [inputs], False
    if isinstance(inputs, list) and len(inputs) == 2 and all(isinstance(t, str) for t in inputs):
        return [(inputs[0], inputs[1])], False
    if isinstance(inputs, list) and inputs:
        return [seq(x) for x in inputs], True
    raise TypeError("`inputs` must be a string, a [string, string] pair or a non-empty list of those")


def splade_response(vecs) -> list:
    """TEI's /embed_sparse body: per input, ``[{"index", "value"}]`` of its non-zero words in index order."""
    import numpy as np

    out = []
    for v in vecs:
        nz = np.flatnonzero(v > 0)
        out.append([{"index": int(i), "value": float(v[i])} for i in nz])
    return out


def resolve_pooling(flag: str | None, snapshot_dir: str | None, model_id: str) -> str:
    """The pooling to serve, resolved as TEI resolves it: --pooling when given; else the Pooling module of the snapshot's
    sentence-transformers config (modules.json -> 1_Pooling/config.json); else the model-id table; else cls.  Raises
    ValueError for a --pooling other than cls / mean and for a snapshot that declares a pooling other than those two.
    --pooling splade is served for a masked-LM snapshot and for the SPLADE ids of SPLADE_MODEL_IDS (as TEI, which refuses it
    on a model without an MLM head); anywhere else it is refused like any other pooling."""
    from b200rt.weights import is_masked_lm_dir, pooling_from_dir

    if flag == "splade" and (model_id in SPLADE_MODEL_IDS or (snapshot_dir and is_masked_lm_dir(snapshot_dir))):
        return flag
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
    ap.add_argument("--pooling", default=None, help="cls, mean or splade (a masked-LM model); default: the snapshot's sentence-transformers "
                    "Pooling config, else cls")
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
            sd = W.read_safetensors(args.weights)
            if "classifier.weight" in sd:  # a BertForSequenceClassification checkpoint
                cfg_path = os.path.join(os.path.dirname(os.path.abspath(args.weights)), "config.json")
                cfg = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
                return W.load_hf_classifier(sd, cfg) + (f"safetensors {args.weights}",)
            return W.load_safetensors(args.weights) + (f"safetensors {args.weights}",)
        if os.path.isdir(args.weights):
            if W.is_nomic_dir(args.weights):
                return W.load_hf_nomic_dir(args.weights) + (f"nomic-bert directory {args.weights}",)
            return W.load_hf_dir(args.weights) + (f"HF directory {args.weights}",)
        return geometry_for_model_id(args.model_id), np.fromfile(args.weights, np.float32), f"flat blob {args.weights}"
    cache = args.huggingface_hub_cache or os.environ.get("HUGGINGFACE_HUB_CACHE") or os.environ.get("HF_HUB_CACHE")
    if cache:
        snap = W.resolve_hub_snapshot(cache, args.model_id)
        if snap:
            if W.is_nomic_dir(snap):
                return W.load_hf_nomic_dir(snap) + (f"nomic-bert hub snapshot {snap}",)
            return W.load_hf_dir(snap) + (f"hub snapshot {snap}",)
    g = geometry_for_model_id(args.model_id)
    if "num_labels" in g:
        return g, W.random_classifier_blob(g, 0), None
    if "rope_theta" in g:
        return g, W.random_nomic_blob(g, 0), None
    return g, random_blob(geometry=g), None


def load_splade_weights(args):
    """Weights of a SPLADE model: the masked-LM checkpoint the weights directory holds, else (an id of SPLADE_MODEL_IDS with no
    snapshot) seeded random init of bge-base's geometry with a loud notice.  A snapshot without an MLM head is refused."""
    from b200rt import weights as W

    d = weights_dir(args)
    if d:
        if not W.is_masked_lm_dir(d):
            raise ValueError(f"--pooling splade needs a masked-LM checkpoint (BertForMaskedLM); {d} has no cls.predictions head")
        return W.load_hf_masked_lm_dir(d) + (f"masked-LM snapshot {d}",)
    g = geometry_for_model_id(args.model_id)
    return g, W.random_splade_blob(g, 0), None


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
        self.splade = self.pooling == "splade"
        geometry, blob, source = load_splade_weights(args) if self.splade else load_weights(args)
        if source is None:
            print(f"[text-embeddings-router/b200] no weights for {args.model_id!r} offline: seeded random init", file=sys.stderr)
        else:
            print(f"[text-embeddings-router/b200] weights: {source}", file=sys.stderr)
        print(f"[text-embeddings-router/b200] pooling: {self.pooling}", file=sys.stderr)
        self.geometry = geometry
        self.classifier = "num_labels" in geometry
        if self.classifier:
            from b200rt.weights import default_id2label

            self.id2label = geometry.get("id2label") or default_id2label(geometry["num_labels"])
            kind = "reranker" if geometry["num_labels"] == 1 else "classifier"
            print(f"[text-embeddings-router/b200] {kind}: BertForSequenceClassification, {geometry['num_labels']} label(s)"
                  + (" -- SEEDED weights, scores are not the real model's" if source is None else ""), file=sys.stderr)
            self.model = b200rt.ClassifierModel(geometry, blob)
        elif self.splade:
            print("[text-embeddings-router/b200] SPLADE: BertForMaskedLM, sparse vectors over the vocabulary through /embed_sparse"
                  + (" -- SEEDED weights, vectors are not the real model's" if source is None else ""), file=sys.stderr)
            self.model = b200rt.SparseEmbedModel(geometry, blob)
        elif self.long_context:
            print(f"[text-embeddings-router/b200] nomic-bert: rotary positions, inputs up to {geometry['max_pos']} tokens"
                  + (" -- SEEDED weights, vectors are not the real model's" if source is None else ""), file=sys.stderr)
            self.model = b200rt.NomicEmbedModel(geometry, blob, pooling=self.pooling)
        else:
            self.model = b200rt.EmbedModel(geometry, blob, pooling=self.pooling)
        self.n_gpus = n_gpus

    def embed(self, inputs, truncate: bool = False):
        np = self.np
        rows = [self.tok.encode(t, self.geometry["max_pos"], truncate or self.args.auto_truncate) for t in inputs]
        lens = np.array([len(r) for r in rows], np.int32)
        ids = np.zeros((len(rows), int(lens.max())), np.int32)
        for i, r in enumerate(rows):
            ids[i, : len(r)] = r
        return self.model.embed(ids, lens)

    def classify(self, inputs, truncate: bool):
        """``[n, num_labels]`` raw logits of strings and (text, text) pairs; ValueError when one is too long (TEI: 413)."""
        np = self.np
        n = self.geometry["max_pos"]
        rows, segs = [], []
        for x in inputs:
            if isinstance(x, tuple):
                r, sg = self.tok.encode_pair(x[0], x[1], n, truncate)
            else:
                r = self.tok.encode(x, n, truncate)
                sg = len(r)
            rows.append(r)
            segs.append(sg)
        lens = np.array([len(r) for r in rows], np.int32)
        ids = np.zeros((len(rows), int(lens.max())), np.int32)
        for i, r in enumerate(rows):
            ids[i, : len(r)] = r
        return self.model.classify(ids, lens, np.array(segs, np.int32))

    @property
    def long_context(self) -> bool:
        """A nomic-bert model (kind "nomic_bert"): inputs up to its max_pos, up to 8192 tokens."""
        return "rope_theta" in self.geometry

    def info(self) -> dict:
        """TEI's /info.  An embedding model's is what it always was; a classifier's reports model_type as TEI does."""
        args = self.args
        d = {"model_id": args.model_id, "model_dtype": "float16", "max_client_batch_size": args.max_client_batch_size,
             "max_input_length": self.geometry["max_pos"] if self.long_context else GEOMETRY["max_pos"],
             "backend": f"b200rt x{self.n_gpus}"}
        if not self.classifier:
            d["pooling"] = self.pooling
            return d
        labels = {str(k): v for k, v in sorted(self.id2label.items())}
        kind = "reranker" if self.geometry["num_labels"] == 1 else "classifier"
        d["model_type"] = {kind: {"id2label": labels, "label2id": {v: int(k) for k, v in labels.items()}}}
        return d


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
                self._send(200, engine.info())
            else:
                self._send(404, {"error": "not found", "error_type": "NotFound"})

        def _rerank(self, req):
            query, texts = req.get("query"), req.get("texts")
            if not isinstance(query, str) or not isinstance(texts, list) or not texts or not all(isinstance(t, str) for t in texts):
                raise TypeError("`query` must be a string and `texts` a non-empty list of strings")
            return query, texts

        def do_POST(self):
            if self.path in ("/rerank", "/predict"):
                return self._classify()
            if self.path == "/embed_sparse":
                return self._embed(sparse=True)
            if self.path not in ("/embed", "/"):
                return self._send(404, {"error": "not found", "error_type": "NotFound"})
            return self._embed(sparse=False)

        def _embed(self, sparse: bool):
            if engine.classifier:
                return self._send(400, {"error": f"{engine.args.model_id} is a classifier: use /rerank or /predict", "error_type": "Backend"})
            if engine.splade and not sparse:
                return self._send(400, {"error": f"{engine.args.model_id} is a SPLADE model: use /embed_sparse", "error_type": "Backend"})
            if sparse and not engine.splade:
                return self._send(400, {"error": f"{engine.args.model_id} is not a SPLADE model: use /embed", "error_type": "Backend"})
            try:
                req = json.loads(self.rfile.read(int(self.headers.get("Content-Length", "0"))))
                inputs = req["inputs"]
                if isinstance(inputs, str):
                    inputs = [inputs]
                if not isinstance(inputs, list) or not inputs or not all(isinstance(t, str) for t in inputs):
                    raise TypeError("`inputs` must be a string or a non-empty list of strings")
                # TEI's `truncate`: honoured by /embed_sparse and by the long-context kind; other models' /embed answers stay as
                # they were (413 past max_pos unless --auto-truncate)
                truncate = bool(req.get("truncate", False)) if sparse or engine.long_context else False
            except Exception as e:  # noqa: BLE001
                return self._send(422, {"error": f"Failed to deserialize the JSON body: {e}", "error_type": "Validation"})
            if len(inputs) > engine.args.max_client_batch_size:
                return self._send(413, {"error": f"batch size {len(inputs)} > maximum allowed batch size {engine.args.max_client_batch_size}",
                                        "error_type": "Validation"})
            try:
                vecs = engine.embed(inputs, truncate)
            except ValueError as e:
                return self._send(413, {"error": str(e), "error_type": "Validation"})
            except Exception as e:  # noqa: BLE001
                return self._send(500, {"error": str(e), "error_type": "Backend"})
            self._send(200, splade_response(vecs) if sparse else vecs.tolist())

        def _classify(self):
            if not engine.classifier:
                return self._send(400, {"error": f"{engine.args.model_id} is an embedding model: use /embed", "error_type": "Backend"})
            rerank = self.path == "/rerank"
            try:
                req = json.loads(self.rfile.read(int(self.headers.get("Content-Length", "0"))))
                if rerank:
                    query, texts = self._rerank(req)
                    inputs, batch = [(query, t) for t in texts], True
                else:
                    inputs, batch = parse_predict_inputs(req.get("inputs"))
            except Exception as e:  # noqa: BLE001
                return self._send(422, {"error": f"Failed to deserialize the JSON body: {e}", "error_type": "Validation"})
            if rerank and engine.geometry["num_labels"] != 1:
                return self._send(400, {"error": "/rerank needs a model with one label (a reranker); use /predict", "error_type": "Backend"})
            if len(inputs) > engine.args.max_client_batch_size:
                return self._send(413, {"error": f"batch size {len(inputs)} > maximum allowed batch size {engine.args.max_client_batch_size}",
                                        "error_type": "Validation"})
            truncate = bool(req.get("truncate", False)) or engine.args.auto_truncate
            raw = bool(req.get("raw_scores", False))
            try:
                logits = engine.classify(inputs, truncate)
            except ValueError as e:
                return self._send(413, {"error": str(e), "error_type": "Validation"})
            except Exception as e:  # noqa: BLE001
                return self._send(500, {"error": str(e), "error_type": "Backend"})
            if rerank:
                return self._send(200, rerank_response(logits, texts, raw, bool(req.get("return_text", False))))
            res = [predict_response(row, engine.id2label, raw) for row in logits]
            self._send(200, res if batch else res[0])

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
