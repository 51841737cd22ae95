#!/usr/bin/env python
"""SPLADE against the CLS embedder on one H100, in one process.  naver/splade-v3's geometry (bge-base, 12 layers, the 30 522-word
vocabulary) and a CLS-pooled bge-base embedder of the same encoder weights run full device-resident waves (b200rt_embed_device
on a torch stream, timed with CUDA events) of the 512-, 128- and 64-token buckets, alternating over >= 2 s windows.  Then, in
a separate profiled run (torch.profiler, CUDA activities), the device time per wave of the head's own kernels and the decoder
GEMM's TFLOP/s from 2 M 30 720 H; and the four head launches by name from the engine's launch events (the transform GEMM
shares its kernel with every layer's FFN1, which the profiler cannot tell apart).  Last, the epilogue's cost: the decoder GEMM (EPI_SPLADE_MAX) against an
EPI_BIAS_F16 GEMM of the same shape, M = 8 192, through the debug entries.  Prints one JSON line; the card's name, power
limit and SM clocks are read in the same run.  Fails without a GPU.

    python tools/splade_bench.py [--windows 4] [--window-s 2.0] [--out FILE]
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
from rerank_bench import kernel_times  # noqa: E402

BUCKETS = (512, 128, 64)
VPAD = 30720
HEAD = ("gemm_mlm_transform", "mlm_ln_stats", "gemm_splade", "splade_finalize")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4, help="timed windows per (model, bucket), alternating")
    ap.add_argument("--window-s", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    a = ap.parse_args()

    import numpy as np
    import torch
    import b200rt
    from b200rt.weights import BGE_BASE_GEOMETRY, blob_numel, random_splade_blob
    from oracle import bge_ref as R

    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the CUDA path only")
    info = card()
    b200rt.init(devices=[0])
    g = BGE_BASE_GEOMETRY
    blob = random_splade_blob(g, 0)
    splade = b200rt.SparseEmbedModel(g, blob)
    embedder = b200rt.EmbedModel(g, blob[:blob_numel(g)])  # the same encoder weights, CLS-pooled
    cap_rows = splade.debug_cap_rows()
    ts = torch.cuda.Stream()
    waves, shapes = {}, {}
    for S in BUCKETS:
        B = cap_rows // S
        d_ids = torch.from_numpy(R.synth_ids(B, S, seed=S)).cuda()
        d_lens = torch.full((B,), S, dtype=torch.int32, device="cuda")
        d_sp = torch.empty((B, g["vocab"]), dtype=torch.float32, device="cuda")
        d_em = torch.empty((B, g["hidden"]), dtype=torch.float32, device="cuda")
        shapes[S] = B

        def run(model, out, d_ids=d_ids, d_lens=d_lens, B=B, S=S):
            return lambda: model.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), B, S, out.data_ptr(), ts.cuda_stream)

        waves[f"splade_{S}"] = run(splade, d_sp)
        waves[f"cls_{S}"] = run(embedder, d_em)

    per_window = {}
    for name, wave in waves.items():
        with torch.cuda.stream(ts):
            for _ in range(3):
                wave()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.cuda.stream(ts):
            for _ in range(5):
                wave()
        torch.cuda.synchronize()
        per_window[name] = max(5, int(a.window_s / ((time.perf_counter() - t0) / 5)) + 1)
    rates = {name: [] for name in waves}
    for _ in range(a.windows):
        for name, wave in waves.items():
            n = per_window[name]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(ts):
                e0.record()
                for _ in range(n):
                    wave()
                e1.record()
            torch.cuda.synchronize()
            rates[name].append(n * shapes[int(name.split("_")[1])] / (e0.elapsed_time(e1) / 1e3))
    items_s = {k: float(np.median(v)) for k, v in rates.items()}

    from torch.profiler import ProfilerActivity, profile

    n_prof = 10
    head = {}
    for S in BUCKETS:
        wave = waves[f"splade_{S}"]
        with torch.cuda.stream(ts):
            wave()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with torch.cuda.stream(ts):
                for _ in range(n_prof):
                    wave()
            torch.cuda.synchronize()
        kt = kernel_times(prof, n_prof)
        pick = lambda *keys: sum(v for k, v in kt.items() if all(s in k for s in keys))  # noqa: E731
        M = shapes[S] * S
        # the transform GEMM shares its instantiation with every layer's FFN1, so the profiler cannot name it: the engine's
        # event timing below does
        h = {
            "mlm_ln_stats_ms": pick("mlm_ln_stats_kernel"),
            "gemm_splade_ms": pick("gemm_kernel<4, 256, 6>"),
            "splade_finalize_ms": pick("splade_finalize_kernel"),
            "wave_ms": sum(kt.values()),
        }
        h["gemm_splade_tflops"] = 2.0 * M * VPAD * g["hidden"] / (h["gemm_splade_ms"] / 1e3) / 1e12
        h["head_launches_share_of_wave"] = (h["mlm_ln_stats_ms"] + h["gemm_splade_ms"] + h["splade_finalize_ms"]) / h["wave_ms"]
        head[S] = h
    # per-launch ms of the head from the engine's own event timing (one event between launches), which names each launch
    prof_fwd = {S: {k: v for k, v in splade.profile_forward(shapes[S], S, iters=5).items() if k in HEAD} for S in BUCKETS}

    # the epilogue's cost at one shape: EPI_SPLADE_MAX against EPI_BIAS_F16, M = 8192 rows (16 items of 512), N = 30 720, K = 768
    rng = np.random.default_rng(0)
    Mg, K = 8192, g["hidden"]
    u = rng.standard_normal((Mg, K)).astype(np.float16)
    stats = np.zeros((Mg, K // 128, 2), np.float32)
    stats[..., 1] = 127.0  # unit variance per slice
    w = (rng.standard_normal((VPAD, K)) / np.sqrt(K)).astype(np.float16)
    c = np.zeros(VPAD, np.float32)
    _, ms_bias = b200rt.debug_gemm(0, u, w, c, iters=20, ln_stats=stats)
    _, ms_splade = b200rt.debug_gemm_splade(u, w[: g["vocab"]], c, stats, np.full(Mg // 512, 512, np.int32), 512, VPAD, 1e-12, iters=20)
    flop = 2.0 * Mg * VPAD * K
    epi = {"M": Mg, "N": VPAD, "K": K, "epi_bias_f16_ms": ms_bias, "epi_splade_max_ms": ms_splade,
           "epi_bias_f16_tflops": flop / (ms_bias / 1e3) / 1e12, "epi_splade_max_tflops": flop / (ms_splade / 1e3) / 1e12,
           "splade_over_bias": ms_splade / ms_bias}
    info_after = card()
    res = {
        "metric": "SPLADE (bge-base, 12 layers) vs CLS bge-base, one H100: device-resident items/s per bucket, head kernel ms",
        "card": info, "card_after": info_after, "wave_items": {str(k): v for k, v in shapes.items()},
        "items_per_s": items_s, "items_per_s_windows": rates,
        "splade_over_cls": {str(S): items_s[f"splade_{S}"] / items_s[f"cls_{S}"] for S in BUCKETS},
        "head_profiler_ms_per_wave": {str(k): v for k, v in head.items()},
        "head_event_ms_per_wave": {str(k): v for k, v in prof_fwd.items()},
        "epilogue": epi,
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    b200rt.shutdown()


if __name__ == "__main__":
    main()
