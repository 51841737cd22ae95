"""GPU: every text kind through more than one replica, bitwise the one-replica runtime.

A wave of G replicas is scattered by the root (ids, lens and, for a classifier, segment starts into each replica's slot
buffers), every replica runs its forward on its own items and its last kernel writes its rows into the root's gather buffer
at item_begin[g] * out_dim.  What that adds per kind, and where it has gone wrong before it runs here:

  * a classifier's segment starts on peers (an item submitted without them falls back to its length), and its rows of 1 or
    2 logits; SPLADE's rows of 30 522 words and each replica's own maxima buffer; nomic-bert's per-replica rotary table and
    gate / up interleave, and its long buckets (8 items of 8192 tokens per replica);
  * the split runtime's launch widths for every kernel the kinds use: SPLIT_SMS(k) puts two replicas on one GPU, GEMMs on
    132 - k SMs, attention on k (k = 21: 111 / 21, k = 66: 66 / 66).

Runtimes, each built in turn (the module's own runtime is shut down for the duration and restarted afterwards): one replica
(the baseline), SPLIT_SMS(21), SPLIT_SMS(66), and a pool of min(visible, 8) GPUs (the baseline again on a one-GPU machine).
Every runtime loads the same seeded 2-layer models and runs the same seeded workloads; every result must be bitwise the
baseline's.  The single-bucket tickets run one at a time first, and each one's peer_bytes must be what the dispatcher's
scatter plan predicts (engine.cu, dispatcher_main): replica g != 0's items x (4 S + 4 + 4 [classifier] + 4 out_dim).  That
shows that the split happened and that the gather and its accounting used the kind's out_dim.  A few baseline items are
checked against the kinds' fp64 oracles at the bars of their own test files, so the bitwise comparison is not against a
wrong answer."""
import threading

import numpy as np
import pytest

import clip_text_refs as T
import nomic_refs as N
import rerank_refs as RR
import splade_refs as SR
import test_gpu_bge_large as GL
import test_gpu_clip_text as GC
import test_gpu_forward_chain as FC
import test_gpu_rerank as GR
import test_gpu_splade as GS
from oracle import bge_ref as R

gpu = pytest.mark.gpu

MIN_ITEMS_PER_REPLICA = 8  # engine.cu
MINILM = dict(hidden=384, heads=12, inter=1536)
CLIP_EOS = 49407


def _visible():
    import torch

    return torch.cuda.device_count()


# ------------------------------------------------------------------------------------------------ models and workloads

def _kinds():
    """kind -> (geometry, flat weights, loader(rt) -> model).  All 2 layers, `trained`-style weights."""
    large = GL.mlg.geometry(2)
    base = R.BertGeometry(layers=2)
    minilm = R.BertGeometry(layers=2, **MINILM)
    clip = T.geometry(layers=2, eos_id=CLIP_EOS)
    nomic = N.geometry(layers=2, max_pos=8192)
    k = {}
    f = R.make_weights(large, 31, "trained")
    k["bge_large"] = (large, f, lambda rt, f=f: rt.EmbedModel(R.geometry_dict(large), R.pack_blob(f, large)))
    f = T.make_weights(clip, 32, "trained")
    k["clip_text"] = (clip, f, lambda rt, f=f: rt.ClipTextModel(clip, T.pack_blob(f, clip)))
    f = RR.make_classifier_weights(minilm, 33, "trained", 1)
    k["reranker"] = (minilm, f, lambda rt, f=f: rt.ClassifierModel(RR.geometry_dict(minilm, 1), RR.pack_classifier_blob(f, minilm)))
    f = RR.make_classifier_weights(base, 34, "trained", 2)
    k["classifier2"] = (base, f, lambda rt, f=f: rt.ClassifierModel(RR.geometry_dict(base, 2), RR.pack_classifier_blob(f, base)))
    f = SR.make_splade_weights(base, 35, "splade")
    k["splade"] = (base, f, lambda rt, f=f: rt.SparseEmbedModel(R.geometry_dict(base), SR.pack_splade_blob(f, base)))
    f = N.make_weights(nomic, 36, "trained")
    k["nomic"] = (nomic, f, lambda rt, f=f: rt.NomicEmbedModel(nomic, N.pack(f, nomic), pooling="mean"))
    f = R.make_weights(base, 37, "trained")
    k["bge_base"] = (base, f, lambda rt, f=f: rt.EmbedModel(R.geometry_dict(base), R.pack_blob(f, base)))
    return k


CLASSIFIERS = ("reranker", "classifier2")
BERT_RAGGED = [1, 63, 64, 65, 128, 129, 200, 256, 257, 320, 384, 385, 448, 449, 511, 512, 3, 100]
NOMIC_RAGGED = [64, 65, 500, 1000, 2048, 2049, 3000, 4097, 6000, 8192, 1, 129, 7777]


def _ticket(kind, lens, S, seed, pairs=False):
    """One ticket's inputs: dict(ids, lens[, segs]) of the kind's token ids, [n, S]."""
    lens = np.asarray(lens, np.int32)
    rng = np.random.default_rng(seed)
    if kind == "clip_text":
        return dict(ids=T.synth_ids(lens, S, seed), lens=lens)
    if kind == "nomic":
        ids = np.zeros((len(lens), S), np.int32)
        for i, n in enumerate(lens):
            ids[i, :n] = rng.integers(1000, 30528, n)
        return dict(ids=ids, lens=lens)
    if kind in CLASSIFIERS:
        segs = np.array([rng.integers(1, n + 1) if pairs else n for n in lens], np.int32)
        ids, lens, segs = RR.synth_pairs(lens, segs, S, seed)
        return dict(ids=ids, lens=lens, segs=segs)
    ids, lens = FC.ragged_batch(lens, S, seed)
    return dict(ids=ids, lens=lens)


def _workloads():
    """kind -> {name: ticket}.  "single*": one 64-token length bucket (S - 63 ... S tokens), one at a time, predicted peer
    bytes; the rest: ragged tickets
    over every bucket the kind has; "one": the item of 2 G + 1 consecutive one-item calls."""
    rng = np.random.default_rng(5)
    w = {}
    for i, kind in enumerate(("bge_large", "reranker", "classifier2", "splade", "bge_base")):
        S = 256 if kind == "classifier2" else 128
        w[kind] = {
            "single": _ticket(kind, rng.integers(S - 63, S + 1, 40), S, 100 + i, pairs=True),
            "ragged": _ticket(kind, BERT_RAGGED, 512, 200 + i, pairs=True),
            "one": _ticket(kind, [77], 77, 300 + i, pairs=True),
        }
    w["clip_text"] = {"single": _ticket("clip_text", rng.integers(65, 78, 40), 77, 110),
                      "ragged": _ticket("clip_text", [1, 2, 40, 64, 65, 77, 30, 76], 77, 210),
                      "one": _ticket("clip_text", [20], 77, 310)}
    # items travel in 64-token buckets: 8129 ... 8192 tokens is the 8192 bucket (8 items per replica, a full workspace each)
    w["nomic"] = {"single_8192": _ticket("nomic", rng.integers(8129, 8193, 16), 8192, 120),
                  "single_2048": _ticket("nomic", rng.integers(1985, 2049, 40), 2048, 121),
                  "ragged": _ticket("nomic", NOMIC_RAGGED, 8192, 220),
                  "one": _ticket("nomic", [1500], 1536, 320)}
    for i, kind in enumerate(CLASSIFIERS):
        S = 256 if kind == "classifier2" else 128
        # two tickets of one bucket, with and without segment starts: the second's items are single segments (start = len)
        both = _ticket(kind, rng.integers(S - 63, S + 1, 24), S, 130 + i, pairs=True)
        w[kind]["with_segs"] = both
        w[kind]["without_segs"] = dict(ids=both["ids"][::-1].copy(), lens=both["lens"][::-1].copy())
        w[kind]["segs_at_len"] = dict(w[kind]["without_segs"], segs=w[kind]["without_segs"]["lens"].copy())
    # SPLADE: one ticket's rows DMA'd straight into a pinned `out`, another's staged through the slot buffer
    w["splade"]["pinned_out"] = _ticket("splade", rng.integers(65, 129, 24), 128, 140)
    w["splade"]["pageable_out"] = _ticket("splade", rng.integers(65, 129, 24), 128, 141)
    return w


def _submit(model, t, out=None):
    if "segs" in t:
        return model.submit(t["ids"], t["lens"], out=out, segs=t["segs"])
    return model.submit(t["ids"], t["lens"], out=out)


def _call(model, t):
    return model.wait(_submit(model, t)).copy()


def scatter_plan(n, G, rr):
    """The dispatcher's split of one wave of n items (engine.cu, dispatcher_main): (items per replica, the next rotation).
    Everyone when there is enough work, else as many replicas as get MIN_ITEMS_PER_REPLICA items each, starting from a
    rotating one; contiguous ranges of ceil(n / used) items."""
    used = min(G, max(1, n // MIN_ITEMS_PER_REPLICA))
    first = 0 if used == G else rr
    if used != G:
        rr = (rr + used) % G
    per = -(-n // used)
    counts = [0] * G
    for k in range(used):
        counts[(first + k) % G] = min(n, (k + 1) * per) - min(n, k * per)
    return counts, rr


def predicted_peer_bytes(n, S, G, wave_items, out_dim, classifier, rr):
    """(peer bytes, waves, next rotation) of a ticket of n items in one bucket of S tokens, cut into waves of wave_items."""
    total, waves = 0, 0
    per_item = 4 * S + 4 + (4 if classifier else 0) + 4 * out_dim
    while n > 0:
        k = min(n, wave_items)
        counts, rr = scatter_plan(k, G, rr)
        total += sum(counts[1:]) * per_item
        waves += 1
        n -= k
    return total, waves, rr


# ------------------------------------------------------------------------------------------------ one runtime

def _device_entry(rt, model, t, gpu):
    """b200rt_embed_device(_pairs) of the ticket on replica `gpu` (every replica of a split runtime is on device 0)."""
    import torch

    B, S = t["ids"].shape
    d_ids = torch.from_numpy(np.ascontiguousarray(t["ids"])).cuda(0)
    d_lens = torch.from_numpy(t["lens"].copy()).cuda(0)
    d_out = torch.empty((B, model.out_dim), dtype=torch.float32, device="cuda:0")
    if "segs" in t:
        d_segs = torch.from_numpy(t["segs"].copy()).cuda(0)
        model.embed_device(gpu, d_ids.data_ptr(), d_lens.data_ptr(), B, S, d_out.data_ptr(), 0, d_segs=d_segs.data_ptr())
    else:
        model.embed_device(gpu, d_ids.data_ptr(), d_lens.data_ptr(), B, S, d_out.data_ptr(), 0)
    rt.device_sync(gpu)
    return d_out.cpu().numpy()


def _first(t, n):
    return {k: v[:n].copy() for k, v in t.items()}


def run_runtime(rt, kinds, work, split):
    """Load every kind and run every workload; returns (results {(kind, name): array}, peer checks, G)."""
    G = rt.num_gpus()
    models = {k: load(rt) for k, (_, _, load) in kinds.items()}
    res, peer = {}, {}
    # 1. the single-bucket tickets, one at a time, from a fresh runtime (the rotation starts at replica 0)
    rr = 0
    for kind, wl in work.items():
        m = models[kind]
        for name, t in wl.items():
            if not name.startswith("single"):
                continue
            n, S = len(t["lens"]), -(-int(t["lens"].max()) // 64) * 64  # the ticket's one length bucket
            s0 = rt.stats()
            res[kind, name] = _call(m, t)
            s1 = rt.stats()
            pred, waves, rr = predicted_peer_bytes(n, S, G, m.debug_cap_rows() // S * G, m.out_dim, kind in CLASSIFIERS, rr)
            peer[kind, name] = (s1["peer_bytes"] - s0["peer_bytes"], pred, s1["waves"] - s0["waves"], waves)
    # 2. ragged tickets over every bucket, and 2 G + 1 one-item calls (consecutive small waves rotate over the replicas)
    for kind, wl in work.items():
        m = models[kind]
        res[kind, "ragged"] = _call(m, wl["ragged"])
        for i in range(2 * G + 1):
            res[kind, f"one/{i}"] = _call(m, wl["one"])
    # 3. a classifier's tickets with and without segment starts, submitted before either is waited, so that they share a
    #    wave behind four waves of its ragged ticket that hold the slots
    for kind in CLASSIFIERS:
        m, wl = models[kind], work[kind]
        hold = [_submit(m, wl["ragged"]) for _ in range(4)]
        a, b = _submit(m, wl["with_segs"]), _submit(m, wl["without_segs"])
        for h in hold:
            m.wait(h)
        res[kind, "with_segs"], res[kind, "without_segs"] = m.wait(a).copy(), m.wait(b).copy()
        res[kind, "segs_at_len"] = _call(m, wl["segs_at_len"])
    # 4. SPLADE: a pinned `out` (direct D2H) and a pageable one, in one bucket, submitted together
    m, wl = models["splade"], work["splade"]
    pinned = rt.PinnedBuffer((len(wl["pinned_out"]["lens"]), m.out_dim), np.float32)
    try:
        a = _submit(m, wl["pinned_out"], out=pinned.array)
        b = _submit(m, wl["pageable_out"])
        m.wait(a)
        res["splade", "pinned_out"] = pinned.array.copy()
        res["splade", "pageable_out"] = m.wait(b).copy()
    finally:
        pinned.free()
    # 5. the device-resident entry on replica 1 against replica 0 (split runtimes: both replicas on device 0)
    if split:
        for kind, name, n in (("splade", "single", 40), ("classifier2", "single", 40), ("reranker", "single", 40),
                              ("nomic", "single_2048", 8)):
            t = _first(work[kind][name], n)
            for gpu in (0, 1):
                res[kind, f"device{gpu}/{name}"] = _device_entry(rt, models[kind], t, gpu)
    # 6. last: one thread per model, its workload's tickets submitted in a loop and then waited, all models at once
    mixed, errors = {}, []

    def worker(kind):
        try:
            m = models[kind]
            names = [n for n in work[kind] if not n.startswith("one")]
            tickets = [(n, _submit(m, work[kind][n])) for n in names]
            for n, tk in tickets:
                mixed[kind, f"mixed/{n}"] = m.wait(tk).copy()
        except Exception as e:  # noqa: BLE001 -- reported below with the kind
            errors.append((kind, e))

    threads = [threading.Thread(target=worker, args=(k,)) for k in models]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    res.update(mixed)
    return res, peer, G


RUNTIMES = ("one replica", "split 21", "split 66", "pool")


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


@pytest.fixture(scope="module")
def runs(rt):
    """({runtime: (results, peer checks, G)} for RUNTIMES, the kinds, the workloads)."""
    kinds, work = _kinds(), _workloads()
    out = {}
    rt.shutdown()
    try:
        for name in RUNTIMES:
            if name == "one replica":
                rt.init(devices=[0])
            elif name.startswith("split"):
                rt.init(devices=[0], flags=rt.SPLIT_SMS(int(name.split()[1])))
            else:
                rt.init(min(_visible(), 8))
            try:
                out[name] = run_runtime(rt, kinds, work, name.startswith("split"))
            finally:
                rt.shutdown()
            print(f"{name}: {out[name][2]} replicas")
        if out["pool"][2] == 1:
            print("one GPU visible: the pool runtime is the one-replica runtime; the split runtimes carry the multi-replica cases")
    finally:
        rt.init(devices=[0])
    return out, kinds, work


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------ assertions

@gpu
@pytest.mark.parametrize("runtime", RUNTIMES[1:])
def test_every_result_is_bitwise_the_one_replica_runtimes(runs, runtime):
    out, _, _ = runs
    base = out["one replica"][0]
    res, _, G = out[runtime]
    if runtime.startswith("split"):
        assert G == 2, G
    bad = []
    for (kind, name), got in sorted(res.items()):
        key = name.split("/", 1)[1] if name.startswith(("mixed/", "device")) else name
        ref = base[kind, "one/0" if key.startswith("one") else key]
        if name.startswith("device"):
            ref = ref[:len(got)]
        if not np.array_equal(_bits(got), _bits(ref)):
            diff = np.nonzero((_bits(got) != _bits(ref)).any(1))[0]
            bad.append(f"{kind} {name}: items {diff[:8].tolist()} of {len(ref)} differ")
    print(f"{runtime} ({G} replicas): {len(res)} results, {len(bad)} differ from the one-replica runtime")
    assert not bad, "\n".join(bad)


@gpu
@pytest.mark.parametrize("runtime", RUNTIMES)
def test_items_without_segment_starts_fall_back_to_their_length(runs, runtime):
    res = runs[0][runtime][0]
    for kind in CLASSIFIERS:
        assert np.array_equal(_bits(res[kind, "without_segs"]), _bits(res[kind, "segs_at_len"])), kind


@gpu
@pytest.mark.parametrize("runtime", RUNTIMES)
def test_single_bucket_tickets_split_as_the_scatter_plan_predicts(runs, runtime):
    res, peer, G = runs[0][runtime]
    for (kind, name), (got, pred, waves, pred_waves) in sorted(peer.items()):
        print(f"{runtime}: {kind} {name} ({len(res[kind, name])} items): peer bytes {got} (predicted {pred}), waves {waves} "
              f"(predicted {pred_waves})")
        assert (got, waves) == (pred, pred_waves), (kind, name)
        if G > 1:
            assert got > 0, f"{kind} {name}: replica 0 took every item"


@gpu
def test_device_entry_on_replica_1_is_replica_0s(runs):
    for runtime in ("split 21", "split 66"):
        res = runs[0][runtime][0]
        names = sorted({n.split("/", 1)[1] for k, n in res if n.startswith("device")})
        assert names
        for kind, name in {(k, n.split("/", 1)[1]) for k, n in res if n.startswith("device")}:
            assert np.array_equal(_bits(res[kind, f"device1/{name}"]), _bits(res[kind, f"device0/{name}"])), (runtime, kind)


def _ends(x):
    """The two items at the ends of the batch's range (first output column): a well-spread pair to check."""
    return [int(np.argmin(x[:, 0])), int(np.argmax(x[:, 0]))]


@gpu
def test_one_replica_results_match_the_fp64_oracles(runs):
    """Two items of each kind (two classifier pairs per classifier, nomic items <= 2048 tokens) at the bars of the kinds' own
    test files: classifiers max |err| / spread < test_gpu_rerank.PARITY_BAR; SPLADE rel-L2 and max |err| within
    test_gpu_splade's REL_BAR / ABS_BAR; bge-large rel-L2 <= test_gpu_bge_large.REL_TOL; CLIP text rel-L2 <=
    test_gpu_clip_text.BAR; nomic rel-L2 < nomic_refs.BARS[(2, "mean")]."""
    out, kinds, work = runs
    base = out["one replica"][0]
    for kind in CLASSIFIERS:
        g, flat, _ = kinds[kind]
        t, got = work[kind]["single"], base[kind, "single"]
        i = _ends(got)
        ref = RR.classify_np(flat, t["ids"][i], t["lens"][i], t["segs"][i], g)
        spread = float(ref.max() - ref.min())
        err = float(np.abs(got[i] - ref).max()) / spread
        print(f"{kind} items {i}: max |err| / spread {err:.2e} (bar {GR.PARITY_BAR:g}, spread {spread:.3g})")
        assert err < GR.PARITY_BAR
    g, flat, _ = kinds["splade"]
    t, got = work["splade"]["single"], base["splade", "single"]
    ref = SR.splade_np(flat, t["ids"][:2], t["lens"][:2], g)
    rel, err = R.rel_l2(got[:2], ref), np.abs(got[:2] - ref).max(1)
    print(f"splade items 0, 1: rel-L2 {rel.max():.2e} (bar {GS.REL_BAR:g}), max |err| {err.max():.2e} (bar {GS.ABS_BAR:g})")
    assert rel.max() <= GS.REL_BAR and err.max() <= GS.ABS_BAR
    g, flat, _ = kinds["bge_large"]
    t, got = work["bge_large"]["single"], base["bge_large", "single"]
    rel = R.rel_l2(got[:2], R.forward_np(flat, t["ids"][:2], t["lens"][:2], g))
    print(f"bge_large items 0, 1: rel-L2 {rel.max():.2e} (bar {GL.REL_TOL:g})")
    assert rel.max() <= GL.REL_TOL
    g, flat, _ = kinds["clip_text"]
    t, got = work["clip_text"]["single"], base["clip_text", "single"]
    rel = T.rel_l2(got[:2], T.forward_np(flat, t["ids"][:2], t["lens"][:2], g))
    print(f"clip_text items 0, 1: rel-L2 {rel.max():.2e} (bar {GC.BAR:g})")
    assert rel.max() <= GC.BAR
    g, flat, _ = kinds["nomic"]
    t, got = work["nomic"]["single_2048"], base["nomic", "single_2048"]
    rel = R.rel_l2(got[:2], N.forward_np(flat, t["ids"][:2], t["lens"][:2], g))
    print(f"nomic items 0, 1 (2048 bucket): rel-L2 {rel.max():.2e} (bar {N.BARS[(2, 'mean')]:g})")
    assert rel.max() < N.BARS[(2, "mean")]


# ------------------------------------------------------------------------------------------------ CPU: the plan restated

def test_scatter_plan():
    assert scatter_plan(40, 1, 0) == ([40], 0)
    assert scatter_plan(40, 2, 0) == ([20, 20], 0)
    assert scatter_plan(16, 2, 1) == ([8, 8], 1)
    assert scatter_plan(1, 2, 0) == ([1, 0], 1) and scatter_plan(1, 2, 1) == ([0, 1], 0)
    assert scatter_plan(40, 8, 6) == ([8, 8, 8, 0, 0, 0, 8, 8], 3)  # 5 replicas from 6, wrapping: 6 7 0 1 2
    assert scatter_plan(45, 3, 0) == ([15, 15, 15], 0)
    assert predicted_peer_bytes(16, 8192, 2, 16, 768, False, 0) == (8 * (4 * 8192 + 4 + 4 * 768), 1, 0)
    assert predicted_peer_bytes(40, 2048, 1, 33, 768, False, 0) == (0, 2, 0)
