#!/usr/bin/env python
"""The four bge-base GEMMs of one 132-item, 512-token wave (M = 67 584) through b200rt_debug_gemm, each timed over a >= 1 s
window of back-to-back launches (CUDA events), at 132 and at 66 SMs.  Per shape and width: ms per launch, algorithmic
TFLOP/s, the operand bytes TMA moves from L2 into shared memory per launch -- computed from the shapes and the cluster
size: every CTA loads its A [128 x 64] per k-block, and a cluster of `cm` CTAs loads the W [BN x 64] it shares once --
that traffic over the time, and the CTAs launched.  The card's name, power limit and SM clock are read in the same run,
the clock as the lowest of the samples taken during each window (fewer SMs draw less power and may clock higher).  Prints
one JSON line.

    python tools/gemm_probe.py [--cm 2] [--root DIR] [--window-s 1.0] [--out FILE]

--root loads the b200rt package of another checkout (an earlier build, for a before / after pair; give --cm 1 for a
build whose GEMM is not clustered).
"""
import argparse
import inspect
import json
import os
import sys
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from bge_small_bench import card  # noqa: E402

M = 132 * 512
SHAPES = [  # name, epi, N, K (bge-base; epi 0/1 fold the LayerNorm of K, epi 2 re-applies the one of N)
    ("qkv", 0, 2304, 768),
    ("attn_out", 2, 768, 768),
    ("ffn1", 1, 3072, 768),
    ("ffn2", 2, 768, 3072),
]


def operand_bytes(N, K, cm):
    bn = 256 if N % 256 == 0 else 128
    m_tiles = -(-M // 128)
    pairs = -(-m_tiles // cm) * (N // bn)
    kblocks = K // 64
    return pairs * kblocks * (cm * 128 * 64 * 2 + bn * 64 * 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cm", type=int, default=2, help="CTAs per GEMM cluster of the build that is loaded")
    ap.add_argument("--root", default=ROOT, help="repository whose b200rt package is loaded")
    ap.add_argument("--window-s", type=float, default=1.0)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(a.root, "modal-examples_b200"))
    import numpy as np
    import b200rt

    info = card()
    b200rt.init(devices=[0])
    reports_ctas = "want_ctas" in inspect.signature(b200rt.debug_gemm).parameters
    rng = np.random.default_rng(0)
    result = {"metric": "bge-base GEMMs at M = 67584 (one 132-item, 512-token wave), b200rt_debug_gemm", "card": info,
              "root": os.path.abspath(a.root), "cm": a.cm, "shapes": {}}
    for name, epi, N, K in SHAPES:
        a16 = rng.standard_normal((M, K), dtype=np.float32).astype(np.float16)
        w16 = (rng.standard_normal((N, K), dtype=np.float32) * 0.05).astype(np.float16)
        bias = rng.standard_normal(N, dtype=np.float32)
        ln_w = N if epi == 2 else K
        st = np.stack([np.zeros((M, ln_w // 128), np.float32), np.full((M, ln_w // 128), 128.0, np.float32)], -1)
        kw = dict(ln_stats=st, eps=1e-12)
        if epi == 2:
            kw.update(resid=rng.standard_normal((M, N), dtype=np.float32), ln_gamma=np.ones(N, np.float32),
                      ln_beta=np.zeros(N, np.float32), want_stats=True)
        flop = 2.0 * M * N * K
        nbytes = operand_bytes(N, K, a.cm)
        rows = {}
        for sms in (132, 66):
            extra = dict(want_ctas=True) if reports_ctas else {}
            r = b200rt.debug_gemm(epi, a16, w16, bias, iters=20, sms=sms, **kw, **extra)  # warm-up; sizes the window
            iters = max(20, int(a.window_s / (r[1] / 1e3)) + 1)
            # the call also uploads the operands, so the clock is sampled all through it; the lowest sample is the one under load
            clocks, done = [], threading.Event()

            def sample():
                while not done.wait(0.25):
                    clocks.append(card().get("sm_clock_mhz"))

            t = threading.Thread(target=sample)
            t.start()
            r = b200rt.debug_gemm(epi, a16, w16, bias, iters=iters, sms=sms, **kw, **extra)
            done.set()
            t.join()
            ms = r[1]
            clocks = [c for c in clocks if c is not None]
            rows[str(sms)] = {"ms": ms, "iters": iters, "tflops": flop / (ms * 1e-3) / 1e12,
                              "l2_to_smem_gb": nbytes / 1e9, "l2_to_smem_tb_s": nbytes / (ms * 1e-3) / 1e12,
                              "ctas": r[-1] if reports_ctas else None, "sm_clock_mhz": min(clocks) if clocks else None}
        result["shapes"][name] = {"epi": epi, "N": N, "K": K, **{f"sms_{k}": v for k, v in rows.items()}}
        print(f"{name:8s} N={N:4d} K={K:4d} " + "  ".join(
            f"sms {k}: {v['ms']:.3f} ms {v['tflops']:.0f} TFLOP/s {v['l2_to_smem_tb_s']:.2f} TB/s ctas {v['ctas']} "
            f"clock {v['sm_clock_mhz']} MHz" for k, v in rows.items()), file=sys.stderr)
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    b200rt.shutdown()


if __name__ == "__main__":
    main()
