#!/usr/bin/env python
"""nomic-embed-text (kind "nomic_bert", 12 layers) beside a mean-pooled bge-base embedder on one H100, in one process.  Full
device-resident waves (b200rt_embed_device on a torch stream, timed with CUDA events) of the 512-, 2048- and 8192-token buckets
for nomic and of the 512 bucket for bge-base, alternating over >= 2 s windows; then each launch's time per wave from the
engine's launch events (b200rt_debug_profile_forward); then the streaming attention against attention_kernel<64, 12> on the
same qkv at S = 512 (a full wave, through the debug entries).  TFLOP/s are algorithmic, from shapes: per item and layer,
linear 2 S (H 3H + H H + H 2I + I H) and attention 4 S^2 H.  Prints one JSON line; the card's name, power limit and SM clocks
are read in the same run.  Fails without a GPU.

    python tools/nomic_bench.py [--windows 3] [--window-s 2.0] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "modal-examples_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bge_small_bench import card  # noqa: E402

BUCKETS = (512, 2048, 8192)
H, I, LAYERS = 768, 3072, 12


def flops_per_item(S: int) -> tuple[float, float]:
    """(total, attention) algorithmic FLOP of one S-token item through 12 layers."""
    linear = 2.0 * S * (H * 3 * H + H * H + H * 2 * I + I * H)
    attn = 4.0 * S * S * H
    return LAYERS * (linear + attn), LAYERS * attn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=3, help="timed windows per wave shape, alternating")
    ap.add_argument("--window-s", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    a = ap.parse_args()

    import numpy as np
    import torch
    import b200rt
    from b200rt.weights import BGE_BASE_GEOMETRY, NOMIC_EMBED_TEXT_GEOMETRY, random_blob, random_nomic_blob

    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the CUDA path only")
    info = card()
    b200rt.init(devices=[0])
    nomic = b200rt.NomicEmbedModel(NOMIC_EMBED_TEXT_GEOMETRY, random_nomic_blob(NOMIC_EMBED_TEXT_GEOMETRY, 0), pooling="mean")
    bge = b200rt.EmbedModel(BGE_BASE_GEOMETRY, random_blob(BGE_BASE_GEOMETRY, 0), pooling="mean")
    cap_rows = nomic.debug_cap_rows()
    ts = torch.cuda.Stream()
    rng = np.random.default_rng(0)
    waves, items = {}, {}
    keep = []
    for name, model, S in [("nomic", nomic, s) for s in BUCKETS] + [("bge_base", bge, 512)]:
        B = cap_rows // S
        d_ids = torch.from_numpy(rng.integers(1000, 30000, (B, S)).astype(np.int32)).cuda()
        d_lens = torch.full((B,), S, dtype=torch.int32, device="cuda")
        d_out = torch.empty((B, H), dtype=torch.float32, device="cuda")
        keep += [d_ids, d_lens, d_out]
        key = f"{name}_{S}"
        items[key] = (B, S)
        waves[key] = (lambda m=model, B=B, S=S, d_ids=d_ids, d_lens=d_lens, d_out=d_out:
                      m.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), B, S, d_out.data_ptr(), ts.cuda_stream))

    per_wave = {}
    for key, wave in waves.items():  # warm-up, and how many waves fill a window
        with torch.cuda.stream(ts):
            for _ in range(2):
                wave()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.cuda.stream(ts):
            wave()
        torch.cuda.synchronize()
        per_wave[key] = time.perf_counter() - t0
    samples = {k: [] for k in waves}
    for _ in range(a.windows):
        for key, wave in waves.items():
            n = max(2, int(a.window_s / max(per_wave[key], 1e-4)))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(ts):
                e0.record(ts)
                for _ in range(n):
                    wave()
                e1.record(ts)
            e1.synchronize()
            samples[key].append(e0.elapsed_time(e1) / n)
    res = {"card": info, "waves": {}}
    for key, ms in samples.items():
        B, S = items[key]
        ms_med = float(np.median(ms))
        total, attn = flops_per_item(S) if key.startswith("nomic") else (None, None)
        res["waves"][key] = {"items": B, "tokens": S, "ms_per_wave": ms_med, "ms_spread": [float(min(ms)), float(max(ms))],
                             "items_per_s": B / ms_med * 1e3, "tokens_per_s": B * S / ms_med * 1e3}
        if total:
            res["waves"][key].update(gflop_per_item=total / 1e9, attention_share=attn / total, tflops=B * total / ms_med / 1e9)
    res["launch_ms"] = {f"nomic_{S}": nomic.profile_forward(cap_rows // S, S, iters=3) for S in BUCKETS}
    res["launch_ms"]["bge_base_512"] = bge.profile_forward(cap_rows // 512, 512, iters=3)
    # the streaming kernel against the resident one on the same qkv, one full 512-token wave
    B, S = cap_rows // 512, 512
    qkv = (rng.standard_normal((B * S, 3 * H)) * 0.7).astype(np.float16)
    lens = np.full(B, S, np.int32)
    ctx_s, ms_s = b200rt.debug_attention_stream(qkv, lens, B, S, iters=20)
    ctx_r, ms_r = b200rt.debug_attention(qkv, lens, B, S, iters=20)
    res["attention_512"] = {"items": B, "stream_ms": ms_s, "resident_ms": ms_r,
                            "bitwise_equal": bool((ctx_s.view(np.uint16) == ctx_r.view(np.uint16)).all())}
    res["card_after"] = card()
    b200rt.shutdown()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
