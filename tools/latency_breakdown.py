#!/usr/bin/env python
"""Diagnostics: where one 512-token item's time goes -- per-kernel device times of a 1-item forward (events between
launches, no graph), the graph-replayed forward end to end, and the host path around it."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "modal-examples_b200"))
import numpy as np, b200rt
from oracle import bge_ref as R
b200rt.init(1)
g = R.BGE_BASE
model = b200rt.EmbedModel(R.geometry_dict(g), R.pack_blob(R.make_weights(g, 0, "hf"), g))
for B in (1, 4, 16):
    prof = model.profile_forward(B, 512, iters=20)
    print(f"B={B}: per-kernel ms (sum over 12 layers):", {k: round(v, 4) for k, v in prof.items()}, "total", round(sum(prof.values()), 4))
ids = R.synth_ids(16, 512, 0)
pin = b200rt.PinnedBuffer((16, 512), np.int32); pin.array[:] = ids
out = b200rt.PinnedBuffer((16, 768), np.float32)
for B in (1, 4, 16):
    lat = []
    for i in range(400):
        t = time.perf_counter(); model.wait(model.submit(pin.array[:B], None, out=out.array[:B], borrow_ids=True)); lat.append((time.perf_counter() - t) * 1e3)
    lat = sorted(lat[100:]); print(f"B={B}: submit+wait p50 {lat[len(lat)//2]:.3f} ms  p10 {lat[len(lat)//10]:.3f}")
s0 = b200rt.stats()
for i in range(200): model.wait(model.submit(pin.array[:1], None, out=out.array[:1], borrow_ids=True))
s1 = b200rt.stats()
print({k: (s1[k] - s0[k]) / 200 for k in ("stage_us", "dispatch_us", "h2d_scatter_us", "forward_us", "d2h_us")})
