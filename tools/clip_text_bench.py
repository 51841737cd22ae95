#!/usr/bin/env python
"""CLIP text tower throughput on one GPU, device-resident (b200rt_embed_device on replica 0): texts/s at 77-token items and at
16-token items, each a full wave run as the scheduler runs it -- padded to its bucket (128 and 64 tokens), the wave's items
being what one wave of that bucket holds -- in alternating 2 s windows with the ViT-B/16 image tower (submit / wait, 64
images per ticket) in the same process.  Also per-kernel ms of one 77-token wave in the 128-token bucket
(b200rt_debug_profile_forward) and TFLOP/s from the shape-derived work at the bucket length (all rows, padding included):
per layer 2 S (3 H^2 + H^2 + 2 H I) + 4 S^2 H -- 10.07 GFLOP per item at S = 128.  The card name, power limit and SM clock
are read (nvidia-smi --query-gpu) in the same call and printed beside the numbers.  Prints one JSON line.

    python tools/clip_text_bench.py [--layers 12] [--windows 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "modal-examples_b200")]


def flops_per_item(S, layers=12, H=512, I=2048):
    return layers * (2 * S * (3 * H * H + H * H + 2 * H * I) + 4 * S * S * H)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--windows", type=int, default=2)
    a = ap.parse_args()
    import numpy as np
    import torch

    import b200rt
    from b200rt import weights as W

    b200rt.init(devices=[0])
    tg = dict(W.CLIP_TEXT_B16_GEOMETRY, layers=a.layers)
    text = b200rt.ClipTextModel(tg, W.random_clip_text_blob(tg))
    vg = dict(W.CLIP_VIT_B16_GEOMETRY)
    img = b200rt.ImageEmbedModel(vg, W.random_vit_blob(vg))
    cap = text.debug_cap_rows()
    res = {"gpu": gpu_info(), "layers": a.layers}
    cases = {}
    for L, bucket in ((77, 128), (16, 64)):
        n = cap // bucket
        ids = torch.full((n, bucket), 49407, dtype=torch.int32, device="cuda:0")  # <|endoftext|> padding past len
        ids[:, :L] = torch.randint(1000, 49000, (n, L), dtype=torch.int32, device="cuda:0")
        ids[:, 0], ids[:, L - 1] = 49406, 49407
        lens = torch.full((n,), L, dtype=torch.int32, device="cuda:0")
        out = torch.empty((n, 512), dtype=torch.float32, device="cuda:0")
        cases[L] = (n, bucket, ids, lens, out)
    px = np.random.default_rng(0).standard_normal((64, 3, 224, 224), dtype=np.float32)

    def text_window(L, secs=2.0):
        n, S, ids, lens, out = cases[L]
        s = torch.cuda.current_stream().cuda_stream
        text.embed_device(0, ids.data_ptr(), lens.data_ptr(), n, S, out.data_ptr(), s)
        torch.cuda.synchronize()
        waves, t0 = 0, time.perf_counter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        while time.perf_counter() - t0 < secs:
            for _ in range(4):
                text.embed_device(0, ids.data_ptr(), lens.data_ptr(), n, S, out.data_ptr(), s)
            waves += 4
            torch.cuda.synchronize()
        e1.record()
        torch.cuda.synchronize()
        return n * waves / (e0.elapsed_time(e1) / 1e3)

    def image_window(secs=2.0):
        img.embed(px)
        k, t0 = 0, time.perf_counter()
        while time.perf_counter() - t0 < secs:
            img.embed(px)
            k += 64
        return k / (time.perf_counter() - t0)

    rates = {77: [], 16: [], "img": []}
    for _ in range(a.windows):
        for L in (77, 16):
            rates[L].append(text_window(L))
            rates["img"].append(image_window())
    for L, bucket in ((77, 128), (16, 64)):
        r = float(np.median(rates[L]))
        res[f"texts_per_s_{L}tok"] = round(r, 1)
        res[f"wave_items_{L}tok"] = cases[L][0]
        res[f"bucket_{L}tok"] = bucket
        res[f"tflops_{L}tok"] = round(r * flops_per_item(bucket, a.layers) / 1e12, 2)
    res["images_per_s_interleaved"] = round(float(np.median(rates["img"])), 1)
    res["gflop_per_item_bucket128"] = round(flops_per_item(128, a.layers) / 1e9, 2)
    res["kernel_ms_77tok_wave"] = {k: round(v, 4) for k, v in text.profile_forward(cases[77][0], 128, iters=3).items()}
    res["gpu_after"] = gpu_info()
    b200rt.shutdown()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
