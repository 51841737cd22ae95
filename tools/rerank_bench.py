#!/usr/bin/env python
"""The cross-encoder against the embedder on one H100, in one process.  cross-encoder/ms-marco-MiniLM-L-6-v2's geometry
(hidden 384, 6 layers, one logit) and the mean-pooled all-MiniLM-L6-v2 embedder (the same encoder) run full waves of the
256-token bucket -- where query + passage pairs land -- device-resident (b200rt_embed_device[_pairs] on a torch stream, timed
with CUDA events), alternating over >= 2 s windows: the wave holds the runtime's 512-token capacity, 2 x 132 = 264 pairs on
an H100 SXM.  Then, in a separate profiled run (torch.profiler, CUDA activities), each kernel's device time per wave: the
classifier's head (cls_head) against the embedder's mean pool, and embed with segments (the pairs' wave) against embed
without (the same wave with one segment per item).  Prints one JSON line; the card's name, power limit and SM clocks are
read in the same run.  Fails without a GPU.

    python tools/rerank_bench.py [--windows 4] [--window-s 2.0] [--out FILE]
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

SEQ = 256
QUERY = 24  # tokens of [CLS] query [SEP]: the passage (token type 1) fills the rest


def kernel_times(prof, n_waves):
    """Device ms per wave of each kernel, by (demangled) name."""
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t and ev.key and not ev.key.startswith(("Memcpy", "Memset", "cuda")):
            out[ev.key] = out.get(ev.key, 0.0) + t / 1e3 / n_waves
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4, help="timed windows per model (alternating)")
    ap.add_argument("--window-s", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    a = ap.parse_args()

    import numpy as np
    import torch
    import b200rt
    from b200rt.weights import MINILM_L6_GEOMETRY, MS_MARCO_MINILM_L6_GEOMETRY, random_blob, random_classifier_blob
    from oracle import bge_ref as R

    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the CUDA path only")
    info = card()
    b200rt.init(devices=[0])
    B = b200rt.wave_capacity_items() * 512 // SEQ
    reranker = b200rt.ClassifierModel(MS_MARCO_MINILM_L6_GEOMETRY, random_classifier_blob(MS_MARCO_MINILM_L6_GEOMETRY, 0))
    embedder = b200rt.EmbedModel(MINILM_L6_GEOMETRY, random_blob(MINILM_L6_GEOMETRY, 0), pooling="mean")
    ids = R.synth_ids(B, SEQ, seed=0)
    ids[:, QUERY - 1] = 102
    d_ids = torch.from_numpy(ids).cuda()
    d_lens = torch.full((B,), SEQ, dtype=torch.int32, device="cuda")
    d_segs = torch.full((B,), QUERY, dtype=torch.int32, device="cuda")
    d_out = torch.empty((B, 384), dtype=torch.float32, device="cuda")
    ts = torch.cuda.Stream()
    waves = {
        "reranker_pairs": lambda: reranker.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), B, SEQ, d_out.data_ptr(), ts.cuda_stream,
                                                        d_segs.data_ptr()),
        "embedder_mean": lambda: embedder.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), B, SEQ, d_out.data_ptr(), ts.cuda_stream),
    }
    single = lambda: reranker.embed_device(0, d_ids.data_ptr(), d_lens.data_ptr(), B, SEQ, d_out.data_ptr(), ts.cuda_stream)  # noqa: E731

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
    wave_ms = {name: [] for name in waves}
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
            ms = e0.elapsed_time(e1)
            rates[name].append(n * B / (ms / 1e3))
            wave_ms[name].append(ms / n)

    # kernel times: a separate profiled run of each wave kind
    from torch.profiler import ProfilerActivity, profile

    n_prof = 20
    prof_ms = {}
    for name, wave in list(waves.items()) + [("reranker_single_segment", single)]:
        with torch.cuda.stream(ts):
            wave()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with torch.cuda.stream(ts):
                for _ in range(n_prof):
                    wave()
            torch.cuda.synchronize()
        prof_ms[name] = kernel_times(prof, n_prof)
    info_after = card()

    def pick(d, *keys):
        hits = {k: v for k, v in d.items() if all(s in k for s in keys)}
        assert len(hits) == 1, (keys, list(d))
        return next(iter(hits.values()))

    rr, em, sg = prof_ms["reranker_pairs"], prof_ms["embedder_mean"], prof_ms["reranker_single_segment"]
    head, pool = pick(rr, "cls_head_kernel"), pick(em, "mean_pool_normalize_kernel")
    embed_segs, embed_plain = pick(rr, "embed_kernel<384, true>"), pick(sg, "embed_kernel<384, false>")
    res = {
        "metric": "cross-encoder vs embedder, one H100: device-resident pairs/s at the 256-token bucket and per-kernel device time",
        "card": info, "card_after": info_after, "wave_items": B, "seq": SEQ, "query_tokens": QUERY,
        "pairs_per_s": {k: float(np.median(v)) for k, v in rates.items()},
        "pairs_per_s_windows": rates,
        "wave_ms": {k: float(np.median(v)) for k, v in wave_ms.items()},
        "cls_head_ms_per_wave": head, "cls_head_share_of_wave": head / sum(rr.values()),
        "mean_pool_ms_per_wave": pool, "mean_pool_share_of_wave": pool / sum(em.values()),
        "embed_segs_ms_per_wave": embed_segs, "embed_no_segs_ms_per_wave": embed_plain,
        "embed_segs_over_no_segs": embed_segs / embed_plain,
        "kernel_ms_per_wave": prof_ms,
    }
    res["reranker_over_embedder_pairs_per_s"] = res["pairs_per_s"]["reranker_pairs"] / res["pairs_per_s"]["embedder_mean"]
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    b200rt.shutdown()


if __name__ == "__main__":
    main()
