# ---
# cmd: ["modal", "run", "examples/embed_bge_native.py"]
# ---
# # BGE-base embeddings on the in-box H100 runtime
#
# The reference's `06_gpu_and_ml/embeddings/text_embeddings_inference.py` with the TEI subprocess replaced by the
# b200rt engine: same `@app.cls` / `@modal.enter` / `@modal.method` shape, same `generate_batches()` (batches of 32,
# remainder dropped) and the same `model.embed.map(..., order_outputs=False)` call site.  Items are token-id rows
# (no tokenizer vocabulary is available offline); weights are a flat fp32 blob (`--weights`), or seeded random weights
# of the BGE-base geometry when none is given.
import time

import modal

BATCH_SIZE = 32
SEQ = 512
GEOMETRY = dict(vocab=30522, hidden=768, layers=12, heads=12, inter=3072, max_pos=512, type_vocab=2, eps=1e-12)

app = modal.App("example-bge-native")

with modal.Image.debian_slim().imports():
    import numpy as np


def random_blob(seed: int = 0):
    """HF-default-init weights (normal sigma 0.02, zero bias, unit LayerNorm) in b200rt's blob order."""
    from b200rt.weights import random_blob as rb

    return rb(GEOMETRY, seed)


@app.cls(gpu="H100:8", max_containers=1)
# Batches in flight; the C++ scheduler coalesces them into waves.  The reference allows 20 containers x 10 inputs = 200
# (text_embeddings_inference.py:79-86); one wave of the 8-replica pool is 8 x 132 items = 33 batches of 32 and the scheduler
# wants two to three waves' worth of tickets pending, hence 96 (each a thread blocked in b200rt_wait with the GIL released).
@modal.concurrent(max_inputs=96)
class TextEmbeddings:
    weights: str = modal.parameter(default="")
    n_gpus: int = modal.parameter(default=0)

    @modal.enter()
    def load(self):
        import b200rt
        import torch

        n = self.n_gpus or torch.cuda.device_count()
        b200rt.init(n)
        blob = np.fromfile(self.weights, np.float32) if self.weights else random_blob()
        self.model = b200rt.EmbedModel(GEOMETRY, blob)
        print(f"engine ready on {n} GPU(s)")

    @modal.exit()
    def unload(self):
        import b200rt

        print("stats:", b200rt.stats())
        b200rt.shutdown()

    @modal.method()
    def embed(self, inputs_with_ids):
        ids, rows = zip(*inputs_with_ids)
        vecs = self.model.embed(np.stack(rows))
        return list(zip(ids, vecs))


@app.local_entrypoint()
def main(n_items: int = 8192, weights: str = "", n_gpus: int = 0):
    rng = np.random.default_rng(0)
    tokens = rng.integers(1000, GEOMETRY["vocab"], size=(n_items, SEQ), dtype=np.int32)
    tokens[:, 0], tokens[:, -1] = 101, 102
    data = [(i, tokens[i]) for i in range(n_items)]

    def generate_batches():
        batch = []
        for item in data:
            batch.append(item)
            if len(batch) == BATCH_SIZE:
                yield batch
                batch = []

    model = TextEmbeddings(weights=weights, n_gpus=n_gpus)
    model.embed.remote(data[:BATCH_SIZE])  # cold start outside the timed region
    t0 = time.perf_counter()
    done = 0
    for output_batch in model.embed.map(generate_batches(), order_outputs=False):
        done += len(output_batch)
    dt = time.perf_counter() - t0
    print(f"embedded {done} items in {dt:.2f} s -> {done / dt:.0f} items/s through modal .map()")
