#!/usr/bin/env python
"""Mean pooling against CLS pooling on one H100, in one process.  CLS and mean models of the same all-MiniLM-L6-v2-geometry
weights (hidden 384, 6 layers) are loaded side by side and alternated over >= 2 s device-resident windows of full waves at
512 tokens (b200rt_embed_device on a torch stream, timed with CUDA events); then b200rt_debug_profile_forward gives the pool
launch's device time per wave for both, and for the bge-base geometry (hidden 768) too.  The mean pool reads every valid
row once (hi + lo, 4 bytes per element): its achieved bytes/s is set against the H100 SXM data sheet's 3.35 TB/s.  Prints one
JSON line; the card's name, power limit and SM clocks are read in the same run.

    python tools/mean_pool_probe.py [--windows 4] [--window-s 2.0] [--out FILE]
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

SEQ = 512
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4, help="timed windows per model (alternating)")
    ap.add_argument("--window-s", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    a = ap.parse_args()

    import numpy as np
    import torch
    import b200rt
    from b200rt.weights import BGE_BASE_GEOMETRY, MINILM_L6_GEOMETRY, random_blob
    from oracle import bge_ref as R

    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this probe measures the CUDA path only")
    info = card()
    b200rt.init(devices=[0])
    cap = b200rt.wave_capacity_items()
    mblob = random_blob(MINILM_L6_GEOMETRY, 0)
    bblob = random_blob(BGE_BASE_GEOMETRY, 0)
    models = {
        "minilm-cls": (MINILM_L6_GEOMETRY, b200rt.EmbedModel(MINILM_L6_GEOMETRY, mblob, pooling="cls")),
        "minilm-mean": (MINILM_L6_GEOMETRY, b200rt.EmbedModel(MINILM_L6_GEOMETRY, mblob, pooling="mean")),
        "bge-base-cls": (BGE_BASE_GEOMETRY, b200rt.EmbedModel(BGE_BASE_GEOMETRY, bblob, pooling="cls")),
        "bge-base-mean": (BGE_BASE_GEOMETRY, b200rt.EmbedModel(BGE_BASE_GEOMETRY, bblob, pooling="mean")),
    }
    timed = ("minilm-cls", "minilm-mean")
    d_ids = torch.from_numpy(R.synth_ids(cap, SEQ, seed=0)).cuda()
    d_lens = torch.full((cap,), SEQ, dtype=torch.int32, device="cuda")
    d_out = torch.empty((cap, 768), dtype=torch.float32, device="cuda")
    ts = torch.cuda.Stream()

    def wave(m):
        m.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), cap, SEQ, d_out.data_ptr(), ts.cuda_stream)

    waves_per_window = {}
    for name in timed:
        m = models[name][1]
        with torch.cuda.stream(ts):
            for _ in range(3):
                wave(m)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.cuda.stream(ts):
            for _ in range(5):
                wave(m)
        torch.cuda.synchronize()
        waves_per_window[name] = max(5, int(a.window_s / ((time.perf_counter() - t0) / 5)) + 1)

    rates = {name: [] for name in timed}
    for _ in range(a.windows):
        for name in timed:
            m, n = models[name][1], waves_per_window[name]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(ts):
                e0.record()
                for _ in range(n):
                    wave(m)
                e1.record()
            torch.cuda.synchronize()
            rates[name].append(n * cap / (e0.elapsed_time(e1) / 1e3))
    info_after = card()

    result = {"metric": "mean vs CLS pooling: device-resident items/s at 512 tokens and the pool launch's device time, one H100",
              "card": info, "card_after": info_after, "wave_items": cap, "seq": SEQ, "models": {}}
    for name, (g, m) in models.items():
        per_kernel = m.profile_forward(cap, SEQ, iters=3)  # ms per wave, each kernel summed over the layers
        pool_name = "mean_pool_normalize" if name.endswith("mean") else "pool_normalize"
        fwd = sum(per_kernel.values())
        r = {"pool_ms_per_wave": per_kernel[pool_name], "forward_ms_per_wave": fwd, "pool_share_of_forward": per_kernel[pool_name] / fwd}
        if name.endswith("mean"):
            nbytes = cap * SEQ * g["hidden"] * 4  # hi + lo of every row, fp16 each
            r.update(pool_bytes_read=nbytes, pool_bytes_per_s=nbytes / (per_kernel[pool_name] / 1e3),
                     pool_fraction_of_hbm_peak=nbytes / (per_kernel[pool_name] / 1e3) / HBM_BYTES_PER_S)
        if name in rates:
            med = float(np.median(rates[name]))
            r.update(items_per_s=med, items_per_s_windows=rates[name],
                     window_spread=(max(rates[name]) - min(rates[name])) / med)
        result["models"][name] = r
    mm = result["models"]
    result["mean_over_cls_items_per_s"] = mm["minilm-mean"]["items_per_s"] / mm["minilm-cls"]["items_per_s"]
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    b200rt.shutdown()


if __name__ == "__main__":
    main()
