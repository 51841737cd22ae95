# ---
# cmd: ["modal", "run", "examples/embed_clip_native.py"]
# ---
# # CLIP ViT-B/16 image embeddings on the in-box H100 runtime
#
# The reference's `06_gpu_and_ml/embeddings/image_embeddings_infinity.py` with the `infinity_emb` engine replaced by the
# b200rt engine: the same `@app.cls` + `@modal.concurrent` class with an `@modal.enter` that brings the model up, an `embed`
# method that takes one batch and returns `(seconds, n_images)` like the reference's (`:330-350`), and the same
# `embedder.embed.map(batches)` fan-out (`:417-421`).  Inputs are preprocessed pixel arrays (there is no image dataset and no
# PIL/torchvision pipeline offline); weights are seeded random weights of the ViT-B/16 geometry unless `--weights` names a
# flat fp32 blob (`b200rt.weights.load_clip_vision_state_dict` makes one from an HF checkpoint).
import time

import modal

BATCH_SIZE = 100  # the reference's batch_size (image_embeddings_infinity.py:62)
GEOMETRY = dict(image=224, patch=16, hidden=768, layers=12, heads=12, inter=3072, proj=512, eps=1e-5)

app = modal.App("example-clip-native")

with modal.Image.debian_slim().imports():
    import numpy as np


@app.cls(gpu="H100:8", max_containers=1)
@modal.concurrent(max_inputs=32)
class ClipEngine:
    weights: str = modal.parameter(default="")
    n_gpus: int = modal.parameter(default=0)

    @modal.enter()
    def init_engine(self):
        import b200rt
        import torch
        from b200rt.weights import random_vit_blob

        n = self.n_gpus or torch.cuda.device_count()
        b200rt.init(n)
        blob = np.fromfile(self.weights, np.float32) if self.weights else random_vit_blob(GEOMETRY)
        self.model = b200rt.ImageEmbedModel(GEOMETRY, blob)
        print(f"engine ready on {n} GPU(s)")

    @modal.exit()
    def shutdown(self):
        import b200rt

        print("stats:", b200rt.stats())
        b200rt.shutdown()

    @modal.method()
    def embed(self, pixels):
        """One batch of preprocessed images [n, 3, 224, 224] float32 -> (seconds inside the engine, n) as the reference
        returns; the embeddings themselves are in `self.last` for callers that want them."""
        st = time.perf_counter()
        self.last = self.model.embed(pixels)
        return time.perf_counter() - st, len(pixels)


@app.local_entrypoint()
def main(n_images: int = 4096, weights: str = "", n_gpus: int = 0):
    rng = np.random.default_rng(0)
    base = rng.standard_normal((BATCH_SIZE, 3, GEOMETRY["image"], GEOMETRY["image"]), dtype=np.float32)
    batches = [base for _ in range(n_images // BATCH_SIZE)]
    embedder = ClipEngine(weights=weights, n_gpus=n_gpus)
    embedder.embed.remote(base)  # cold start outside the timed region
    t0 = time.perf_counter()
    times, counts = zip(*embedder.embed.map(batches))
    dt = time.perf_counter() - t0
    print(f"embedded {sum(counts)} images in {dt:.2f} s -> {sum(counts) / dt:.0f} images/s through modal .map() "
          f"(mean in-engine batch time {1e3 * sum(times) / len(times):.1f} ms)")
