#!/usr/bin/env python
"""bge-large against bge-base on one H100, in one process: device-resident items/s at 512 tokens, each model at its own full
wave capacity (b200rt_model_wave_capacity_items: 99 bge-large items against 132 bge-base items on an H100 SXM), the models
alternated over >= 2 s windows (b200rt_embed_device on a torch stream, timed with CUDA events, as bench.py's `value` is), then
the per-kernel device times of one full wave of each from b200rt_debug_profile_forward.  Prints one JSON line; the card's name,
power limit and SM clocks are read in the same run, because a rate means nothing without them.

    python tools/bge_large_bench.py [--windows 3] [--window-s 2.0] [--out FILE]
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

from bge_small_bench import card  # noqa: E402  (nvidia-smi query of name, power limit and SM clocks)

SEQ = 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=3, help="timed windows per model (alternating)")
    ap.add_argument("--window-s", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    a = ap.parse_args()

    import numpy as np
    import torch
    import b200rt
    from b200rt.weights import BGE_BASE_GEOMETRY, BGE_LARGE_GEOMETRY, random_blob
    from oracle import bge_ref as R

    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the CUDA path only")
    info = card()
    b200rt.init(devices=[0])
    models = {}
    for name, g in (("bge-base", BGE_BASE_GEOMETRY), ("bge-large", BGE_LARGE_GEOMETRY)):
        m = b200rt.EmbedModel(g, random_blob(g, 0))
        models[name] = (g, m, m.wave_capacity_items())
    cap_max = max(c for _, _, c in models.values())
    d_ids = torch.from_numpy(R.synth_ids(cap_max, SEQ, seed=0)).cuda()
    d_lens = torch.full((cap_max,), SEQ, dtype=torch.int32, device="cuda")
    d_out = torch.empty((cap_max, 1024), dtype=torch.float32, device="cuda")
    ts = torch.cuda.Stream()

    def wave(m, cap):
        m.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), cap, SEQ, d_out.data_ptr(), ts.cuda_stream)

    # warm-up, and the number of waves that fills a window
    waves_per_window = {}
    for name, (g, m, cap) in models.items():
        with torch.cuda.stream(ts):
            for _ in range(3):
                wave(m, cap)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.cuda.stream(ts):
            for _ in range(5):
                wave(m, cap)
        torch.cuda.synchronize()
        per = (time.perf_counter() - t0) / 5
        waves_per_window[name] = max(5, int(a.window_s / per) + 1)

    rates = {name: [] for name in models}
    for _ in range(a.windows):
        for name, (g, m, cap) in models.items():
            n = waves_per_window[name]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(ts):
                e0.record()
                for _ in range(n):
                    wave(m, cap)
                e1.record()
            torch.cuda.synchronize()
            rates[name].append(n * cap / (e0.elapsed_time(e1) / 1e3))
    info_after = card()

    result = {"metric": "device-resident items/s at 512 tokens, one H100, bge-large vs bge-base, each at its full wave capacity",
              "card": info, "card_after": info_after, "seq": SEQ, "models": {}}
    for name, (g, m, cap) in models.items():
        geo = R.BertGeometry(**g)
        flops = geo.flops_per_item(SEQ)
        ips = float(np.median(rates[name]))
        per_kernel = m.profile_forward(cap, SEQ, iters=3)  # ms per wave, each kernel summed over the layers
        result["models"][name] = {"wave_items": cap, "items_per_s": ips, "items_per_s_windows": rates[name], "tokens_per_s": ips * SEQ,
                                  "gflop_per_item": flops / 1e9, "algorithmic_tflops": ips * flops / 1e12,
                                  "per_kernel_ms_per_wave": per_kernel, "forward_ms_per_wave": sum(per_kernel.values())}
    r = result["models"]
    result["tflops_large_over_base"] = r["bge-large"]["algorithmic_tflops"] / r["bge-base"]["algorithmic_tflops"]
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    b200rt.shutdown()


if __name__ == "__main__":
    main()
