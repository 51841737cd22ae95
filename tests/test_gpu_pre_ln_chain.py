"""Pre-LN forward-chain conformance: the CLIP ViT and CLIP text towers' chain checks (tests/test_gpu_forward_chain.py's
VitChain, tests/test_gpu_clip_text.py's ClipTextChain) shown to discriminate, and both towers on "hard" weights.

Pre-LN wiring differs from BERT's where a refactor touches it: the residual epilogues add the raw stream (no statistics in)
and emit the statistics the next fold reads, QKV folds LN1 and FFN1 folds LN2, the text tower runs causal attention over a
128-row zero-padded position table and pools by one of two rules, the ViT runs im2col, vit_embed and vit_pool.  The CPU
tests here emulate both 2-layer forwards with the kernels' rounding (kernel_emul) as `debug_trace` returns them: the
emulations pass the chain checks on "trained" and "hard" weights, and every wiring mutant below fails them.  Each mutant also
prints its end-to-end rel-L2 against the fp64 oracle; those that stay under the model-level bar are asserted to, which
records the bugs only the chain can see.

"hard" weights (oracle/clip_ref.make_weights): massive residual channels on token 0 (and two ViT patch tokens), small
gains on them, an attention sink on key 0, peaked attention, LayerNorm gains ~2.5.  Their statistics are asserted on the
fp64 oracle, HF fp32 agrees with the oracle at 12 layers, and tests/golden/clip{,_text}_hard_golden.npz pin them.

Parity bars of the "hard" style, from the emulated fp16-operand floor (the chain emulations below at 12 layers against the
fp64 oracle, on the golden cases; printed by test_hard_parity_floor):
  ViT: floor 3.6e-4 (VH12) -> HARD_BAR_VIT = 1e-3, the tower's general bar, 2.7x the floor;
  CLIP text: floor 2.2e-3 (HB; HC 1.8e-3) -> HARD_BAR_TEXT = 5e-3, the same 2.3x headroom as the general 2e-3 bar has over
  its 8.8e-4 floor.
The GPU tests carry `@gpu`."""
import hashlib
import importlib.util
import math
import os
import time

import numpy as np
import pytest

import clip_text_refs as T
import kernel_emul as KE
import kernel_refs as KR
import test_gpu_clip_text as CT
import test_gpu_forward_chain as FC
import test_gpu_full_wave_chain as FW
from oracle import clip_ref as C

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", "golden", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


vg = _load("make_clip_hard_golden")
tg = _load("make_clip_text_hard_golden")

HARD_BAR_VIT = 1e-3   # emulated floor 3.6e-4 (module docstring)
HARD_BAR_TEXT = 5e-3  # emulated floor 2.2e-3
BAR = {("vit", "trained"): 1e-3, ("vit", "hard"): HARD_BAR_VIT, ("text", "trained"): CT.BAR, ("text", "hard"): HARD_BAR_TEXT}

TEXT_LENS, TEXT_S = [77, 1, 64, 65, 30, 2], 128


def text_batch():
    """The GPU tests' text batch: ragged in the 128-token bucket, an <|endoftext|> inside len before the last one (item 4),
    and one item of two word ids without special tokens (item 5), where the two pooling rules pick different rows."""
    lens = np.array(TEXT_LENS, np.int32)
    ids = T.synth_ids(lens, TEXT_S, seed=5)
    ids[4, 10:14] = T.EOS
    ids[5, :2] = (523, 9001)
    return ids, lens


def vit_case(style, layers=2, fold=KE.fold_ln32, n=3):
    g = C.VitGeometry(layers=layers)
    flat = C.make_weights(g, 1, style)
    px = C.synth_pixels(n, g, 4)
    return FC.VitChain(flat, g, px, fold)


def text_case(style, eos_id, layers=2, fold=KE.fold_ln32):
    g = T.geometry(layers=layers, eos_id=eos_id)
    flat = T.make_weights(g, 1, style)
    ids, lens = text_batch()
    return CT.ClipTextChain(flat, g, ids, lens, fold)


def oracle(ch):
    if isinstance(ch, FC.VitChain):
        return C.forward_np(ch.flat, ch.pixels, ch.g)
    return T.forward_np(ch.flat, ch.ids[:, :ch.g["max_pos"]], ch.lens, ch.g)  # rows past 77 are padding in the 128 bucket


# ================================================================================================ CPU emulation of the chains

VIT_MUTANTS = ("stale_lo", "resid_ln", "ffn1_pstats0", "qkv_pstats1", "fold_swap", "im2col_hwc", "vit_pos_shift", "vit_pool_row1",
               "guard_row", "foreign_buffer")
TEXT_MUTANTS = ("stale_lo", "resid_ln", "ffn1_pstats0", "qkv_pstats1", "fold_swap", "non_causal", "pool_branch", "pos_unpadded",
                "guard_row", "foreign_buffer")


def _emulate_pre_ln(ch, mutant, n_total, head, attention, pool, keep=True):
    """The traces of a pre-LN forward as `debug_trace` returns them (tests/test_gpu_forward_chain.py's emulate_chain for the
    post-LN one): `head(st, snap)` runs the launches before layer 0, `attention(qkv)` the attention, `pool(st)` the pooled
    output.  keep=False keeps the last trace only (12-layer floors)."""
    f, M, eps = ch.flat, ch.M, float(ch.g.eps if isinstance(ch, FC.VitChain) else ch.g["eps"])
    H, I, L = ch.ao16[0].shape[0], ch.ff1[0][0].shape[0], len(ch.qkv)
    rows = M + FC.GUARD
    f16 = lambda w: np.full((rows, w), 0xFFFF, np.uint16).view(np.float16)  # noqa: E731
    st = dict(yhi=f16(H), ylo=f16(H), qkv=f16(3 * H), ctx=f16(H), ffn=f16(I),
              pstats0=np.full((rows, H // KR.SLICE, 2), 0xFFFFFFFF, np.uint32).view(np.float32),
              pstats1=np.full((rows, H // KR.SLICE, 2), 0xFFFFFFFF, np.uint32).view(np.float32))
    names, traces = [], []

    def snap(name=None, out=None):
        if name:
            names.append(name)
        if keep or out is not None:
            traces.append({**{k: v.copy() for k, v in st.items()}, "out": out, "names": list(names), "n_total": n_total, "M": M,
                           "rows": rows})

    def residual(a, w16, bias, p, st_out):
        kw = dict(ln_stats=st["pstats0"][:M], ln_gamma=f[p + "ln1.g"], ln_beta=f[p + "ln1.b"], eps=eps) if mutant == "resid_ln" else {}
        h, lo, v = KE.emulate_gemm(2, a, w16, bias, resid_hilo=(st["yhi"][:M], st["ylo"][:M]), split=True, **kw)
        st["yhi"][:M] = h
        if mutant != "stale_lo":
            st["ylo"][:M] = lo
        st[st_out][:M] = KE.partials32(v)

    snap()
    head(st, snap)
    for l in range(L):
        p = f"l{l}."
        w16, c = KE.fold_ln32(f[p + "qkv.w"], f[p + "ln2.g"], f[p + "ln2.b"], f[p + "qkv.b"]) if mutant == "fold_swap" else ch.qkv[l]
        stats = "pstats1" if mutant == "qkv_pstats1" and l > 0 else "pstats0"
        st["qkv"][:M] = KE.emulate_gemm(0, st["yhi"][:M], w16, c, ln_stats=st[stats][:M], eps=eps)
        if mutant == "guard_row":
            st["qkv"][M] = st["qkv"][M - 1]
        snap("gemm_qkv")
        st["ctx"][:M] = attention(st["qkv"][:M])
        if mutant == "foreign_buffer":
            st["ffn"][0, :H] = st["ctx"][0]
        snap("attention")
        residual(st["ctx"][:M], ch.ao16[l], f[p + "ao.b"], p, "pstats1")
        snap("gemm_attn_out")
        w16, c = KE.fold_ln32(f[p + "ff1.w"], f[p + "ln1.g"], f[p + "ln1.b"], f[p + "ff1.b"]) if mutant == "fold_swap" else ch.ff1[l]
        st["ffn"][:M] = KE.emulate_gemm(3, st["yhi"][:M], w16, c, ln_stats=st["pstats0" if mutant == "ffn1_pstats0" else "pstats1"][:M],
                                        eps=eps)
        snap("gemm_ffn1_qgelu")
        residual(st["ffn"][:M], ch.ff216[l], f[p + "ff2.b"], p, "pstats0")
        snap("gemm_ffn2")
    name, out = pool(st)
    snap(name, out)
    return traces


def _pool32(x, gamma, beta, proj, eps):
    """The pool kernels in fp32: LayerNorm of the pooled rows, projection, L2 normalisation."""
    return KE.l2_normalise32(KE.ln32(x, gamma, beta, eps) @ np.asarray(proj, np.float32).T)


def emulate_vit_chain(ch, mutant=None, keep=True):
    """The ViT forward: im2col, gemm_patch, vit_embed, 5 launches per layer, vit_pool.  Mutants (besides the shared ones of
    _emulate_pre_ln: stale_lo, resid_ln, ffn1_pstats0, qkv_pstats1, fold_swap, guard_row, foreign_buffer):
      im2col_hwc     each patch flattened in (row, column, channel) order instead of (channel, row, column)
      vit_pos_shift  patch token t reads position row t - 1 (the class token's slot forgotten)
      vit_pool_row1  the pool reads the first patch token instead of the class token"""
    g, f, M, T_ = ch.g, ch.flat, ch.M, ch.S
    eps, B, p = g.eps, ch.B, g.patch

    def head(st, snap):
        cols = FC.im2col_ref(ch.pixels, g)
        if mutant == "im2col_hwc":
            gr = g.grid
            hwc = ch.pixels.reshape(B, 3, gr, p, gr, p).transpose(0, 2, 4, 3, 5, 1).reshape(B, gr * gr, -1)
            cols = np.concatenate([np.zeros((B, 1, 3 * p * p), np.float32), hwc], 1).reshape(M, -1).astype(np.float16)
        st["ffn"].reshape(-1)[:cols.size] = cols.reshape(-1)
        snap("im2col")
        st["ctx"][:M] = KE.emulate_gemm(0, cols, ch.patch16, np.zeros(g.hidden, np.float32))
        snap("gemm_patch")
        tk = np.arange(M) % T_
        prow = np.where(tk == 0, 0, tk - 1) if mutant == "vit_pos_shift" else tk
        src = np.where((tk == 0)[:, None], f["cls"][None, :], st["ctx"][:M].astype(np.float32))
        y = KE.ln32(src + f["pos"][prow], f["pre.g"], f["pre.b"], eps)
        st["yhi"][:M], st["ylo"][:M] = KR.split_hilo(y)
        st["pstats0"][:M] = KE.partials32(y)
        snap("vit_embed")

    def attention(qkv):
        return KE.emulate_attention(qkv, [T_] * B, B, T_)

    def pool(st):
        r = np.arange(B) * T_ + (1 if mutant == "vit_pool_row1" else 0)
        x = st["yhi"][r].astype(np.float32) + st["ylo"][r].astype(np.float32)
        return "vit_pool", _pool32(x, f["post.g"], f["post.b"], f["proj.w"], eps)

    return _emulate_pre_ln(ch, mutant, 5 * g.layers + 4, head, attention, pool, keep)


def emulate_clip_text_chain(ch, mutant=None, keep=True):
    """The CLIP text forward: embed (token + the 128-row zero-padded position table), 5 launches per layer, clip_text_pool by
    the model's eos_id rule.  Mutants (besides the shared ones):
      non_causal    bidirectional attention
      pool_branch   the legacy argmax rule whatever eos_id is
      pos_unpadded  position rows 77-127 of the padded table not zero"""
    g, f, M, S = ch.g, ch.flat, ch.M, ch.S
    eps = g["eps"]

    def head(st, snap):
        pos = ch.pos.copy()
        if mutant == "pos_unpadded":
            pos[g["max_pos"]:] = f["pos"][:pos.shape[0] - g["max_pos"]]
        hi, lo, x = KR.embed_exact(ch.ids.reshape(-1), f["token"], pos[:S], np.zeros(g["hidden"], np.float32), S)
        st["yhi"][:M], st["ylo"][:M], st["pstats0"][:M] = hi, lo, KE.partials32(x)
        snap("embed")

    def attention(qkv):
        return KE.emulate_attention(qkv, ch.lens, ch.B, S, heads=g["heads"], head_dim=g["hidden"] // g["heads"],
                                    causal=mutant != "non_causal")

    def pool(st):
        r = np.arange(ch.B) * S + T.pooled_positions(ch.ids, ch.lens, 2 if mutant == "pool_branch" else g["eos_id"])
        x = st["yhi"][r].astype(np.float32) + st["ylo"][r].astype(np.float32)
        return "clip_text_pool", _pool32(x, f["final.g"], f["final.b"], f["proj.w"], eps)

    return _emulate_pre_ln(ch, mutant, 5 * g["layers"] + 2, head, attention, pool, keep)


def emulate(ch, mutant=None, keep=True):
    return (emulate_vit_chain if isinstance(ch, FC.VitChain) else emulate_clip_text_chain)(ch, mutant, keep)


_cases = {}


def cpu_case(tower, style, eos_id=T.EOS):
    key = (tower, style, eos_id)
    if key not in _cases:
        _cases[key] = vit_case(style) if tower == "vit" else text_case(style, eos_id)
    return _cases[key]


CHAINS = [("vit", "trained", None), ("vit", "hard", None), ("text", "trained", 2), ("text", "trained", T.EOS), ("text", "hard", 2),
          ("text", "hard", T.EOS)]


@pytest.mark.parametrize("tower,style,eos_id", CHAINS)
def test_emulated_pre_ln_chain_passes(tower, style, eos_id):
    """3 images / the 6-item text batch, 2 layers: every launch of the emulated forward passes its check, and the pooled output
    is within the model-level bar of the fp64 oracle."""
    ch = cpu_case(tower, style, eos_id)
    margins = {}
    last = FC.run_chain(f"emulated {tower}/{style}", ch, emulate(ch).__getitem__, margins)
    FC.print_margins(f"emulated {tower}/{style} eos {eos_id}", margins)
    assert last["n_total"] == 5 * 2 + (4 if tower == "vit" else 2)
    rel = C.rel_l2(last["out"], oracle(ch))
    print(f"emulated {tower}/{style}: rel-L2 against the fp64 oracle {rel.max():.3e} (bar {BAR[tower, style]:g})")
    assert rel.max() < BAR[tower, style]


# mutants whose end-to-end error stays under the model-level bar: only the chain checks see them
UNDER_BAR = {("vit", "stale_lo"), ("vit", "guard_row"), ("vit", "foreign_buffer"), ("text", "stale_lo"), ("text", "pos_unpadded"),
             ("text", "guard_row"), ("text", "foreign_buffer")}


@pytest.mark.parametrize("tower,mutant", [("vit", m) for m in VIT_MUTANTS] + [("text", m) for m in TEXT_MUTANTS])
def test_chain_checks_reject_pre_ln_wiring_mutants(tower, mutant):
    """`trained` weights; the text tower with eos_id 49407 (the first-match rule, which pool_branch breaks)."""
    ch = cpu_case(tower, "trained")
    traces = emulate(ch, mutant)
    rel = C.rel_l2(traces[-1]["out"], oracle(ch)).max()
    bar = BAR[tower, "trained"]
    print(f"mutant {tower}/{mutant}: emulated end-to-end rel-L2 against the fp64 oracle {rel:.3e} (bar {bar:g})")
    if (tower, mutant) in UNDER_BAR:
        assert rel < bar
    with pytest.raises(AssertionError) as e:
        FC.run_chain(f"mutant {tower}/{mutant}", ch, traces.__getitem__)
    print(f"mutant {tower}/{mutant}: caught: {str(e.value).splitlines()[0][:160]}")


def test_causal_attention_check_accepts_emulation_and_rejects_mutants():
    """8 heads of 64, causal.  Scores climb by sub-block (as test_attention_check_accepts_emulation_and_rejects_mutants' do),
    so a row's running maximum moves at every sub-block it reads; lens short of S so that the key mask can be off by one in
    either direction."""
    B, S, lens = 2, 192, [150, 100]
    rng = np.random.default_rng(1)
    x = rng.standard_normal((B, S, 3, 8, 64)) * 0.5
    u = rng.standard_normal(64)
    u /= np.linalg.norm(u)
    x[:, :, 0] += 4.0 * np.where(rng.random((B, S, 8, 1)) < 0.6, 1.0, -1.0) * u
    x[:, :, 1] += (12.0 * (np.arange(S) // 64))[None, :, None, None] * u
    qkv = x.reshape(B * S, 3 * 512).astype(np.float16)
    emu = lambda m=None, causal=True: KE.emulate_attention(qkv, lens, B, S, m, heads=8, causal=causal)  # noqa: E731
    T.check_causal_attention("causal attention emulation", emu(), qkv, lens, B, S)
    for m, out in (("mask_plus", emu("mask_plus")), ("mask_minus", emu("mask_minus")), ("no_rescale", emu("no_rescale")),
                   ("non_causal", emu(causal=False))):
        with pytest.raises(AssertionError):
            T.check_causal_attention(f"causal attention mutant {m}", out, qkv, lens, B, S)


# ================================================================================================ CPU: the "hard" style

def _ln(x, g, b, eps):
    d = x - x.mean(-1, keepdims=True)
    return d / np.sqrt((d * d).mean(-1, keepdims=True) + eps) * g + b


def layer_stats(flat, x, l, heads, lens, causal, eps):
    """fp64 internals of layer l on the residual x entering it: (attention probabilities [n, heads, S, S] over the valid
    query rows' mask, the valid query mask [n, S], max |qkv|, max |FFN1 pre-activation|)."""
    W = {k: v.astype(np.float64) for k, v in flat.items()}
    p = f"l{l}."
    n, S, h = x.shape
    dh = h // heads
    qkv = _ln(x, W[p + "ln1.g"], W[p + "ln1.b"], eps) @ W[p + "qkv.w"].T + W[p + "qkv.b"]
    q, k, v = (qkv[..., j * h:(j + 1) * h].reshape(n, S, heads, dh).transpose(0, 2, 1, 3) for j in range(3))
    s = q @ k.transpose(0, 1, 3, 2) / math.sqrt(dh)
    mask = (np.arange(S)[None, :] >= np.asarray(lens)[:, None])[:, None, None, :]
    if causal:
        mask = mask | (np.arange(S)[None, :] > np.arange(S)[:, None])[None, None]
    s = np.where(mask, -np.inf, s)
    e = np.exp(s - s.max(-1, keepdims=True))
    prob = e / e.sum(-1, keepdims=True)
    ctx = (prob @ v).transpose(0, 2, 1, 3).reshape(n, S, h)
    x2 = x + ctx @ W[p + "ao.w"].T + W[p + "ao.b"]
    u = _ln(x2, W[p + "ln2.g"], W[p + "ln2.b"], eps) @ W[p + "ff1.w"].T + W[p + "ff1.b"]
    return prob, np.arange(S)[None, :] < np.asarray(lens)[:, None], np.abs(qkv).max(), np.abs(u).max()


def _hard_towers():
    vgeo = C.VitGeometry(layers=12)
    vflat = C.make_weights(vgeo, 1, "hard")
    px = C.synth_pixels(2, vgeo, 4)
    _, vh = C.forward_np(vflat, px, vgeo, return_hidden=True)
    tgeo = T.geometry(layers=12, eos_id=T.EOS)
    tflat = T.make_weights(tgeo, 1, "hard")
    ids, lens = text_batch()
    ids = ids[:, :77]
    _, th = T.forward_np(tflat, ids, lens, tgeo, return_hidden=True)
    return (("vit", vflat, vh, vgeo.heads, [vgeo.tokens] * 2, False, vgeo.eps, "post."),
            ("text", tflat, th, tgeo["heads"], lens, True, tgeo["eps"], "final."))


def test_hard_style_statistics():
    """On the fp64 oracle, 12 layers, through every layer: the massive channels on token 0 (and the two ViT patch tokens) at
    100-400 and >= 50x the median |x|; a sink (> half the weight on key 0) in >= 15 % of the valid (query, head) rows of every
    layer and >= 25 % over the tower; rows close to one-hot (max p > 0.9) in >= 5 %; small gains on the massive channels, the
    other gains around 2.5, non-zero biases; every residual, QKV and FFN1 value below 2 000."""
    ch = C.HARD_CHANNELS
    for tower, flat, hidden, heads, lens, causal, eps, final in _hard_towers():
        sinks, peaks = [], []
        tokens = [0] + (list(C.HARD_PATCH_TOKENS) if tower == "vit" else [])
        for l, x in enumerate(hidden):
            x = x.astype(np.float64)
            med = np.median(np.abs(x))
            mas = np.abs(x[:, tokens][..., ch])
            assert 100 <= mas.min() and mas.max() <= 400 and mas.min() >= 50 * med, (tower, l, mas.min(), mas.max(), med)
            assert np.abs(x).max() < 2000
            if l == len(hidden) - 1:
                print(f"{tower}: massive channels {mas.min():.0f}-{mas.max():.0f}, median |x| {med:.2f} at the last layer")
                continue
            prob, valid, qkv_max, u_max = layer_stats(flat, x, l, heads, lens, causal, eps)
            vq = np.broadcast_to(valid[:, None, :], prob.shape[:3])
            sinks.append((prob[..., 0] > 0.5)[vq].mean())
            peaks.append((prob.max(-1) > 0.9)[vq].mean())
            assert qkv_max < 2000 and u_max < 2000, (tower, l, qkv_max, u_max)
        print(f"{tower}: sink fraction per layer {np.round(sinks, 2).tolist()}, one-hot fraction {np.round(peaks, 2).tolist()}")
        assert min(sinks) >= 0.15 and np.mean(sinks) >= 0.25 and min(peaks) >= 0.05
        gains = [n for n in flat if n.endswith(".g")]
        for n in gains:
            assert (flat[n][ch] <= 0.05).all() or n == "pre.g", n
            rest = np.delete(flat[n], ch)
            assert 2.0 <= np.median(rest) <= 3.0, (n, np.median(rest))
        for n in flat:
            if n.endswith(".b"):
                assert (flat[n] != 0).mean() > 0.9, n
        assert flat[final + "g"][ch].max() <= 0.05


def test_hard_style_keeps_the_shared_hf_draws():
    """The "hard" branch draws after the shared "hf" draws: every matrix it does not rescale is the "hf" one."""
    g = C.VitGeometry(layers=2)
    hf, hard = C.make_weights(g, 1, "hf"), C.make_weights(g, 1, "hard")
    assert np.array_equal(hf["l1.ao.w"], hard["l1.ao.w"]) and np.array_equal(hf["l0.ff2.w"], hard["l0.ff2.w"])
    tgeo = T.geometry(layers=2)
    hf, hard = T.make_weights(tgeo, 1, "hf"), T.make_weights(tgeo, 1, "hard")
    assert np.array_equal(hf["token"], hard["token"]) and np.array_equal(hf["l1.ff2.w"], hard["l1.ff2.w"])


def test_hf_fp32_agrees_with_the_fp64_oracle_on_hard_weights_at_12_layers():
    g = C.VitGeometry(layers=12)
    flat = C.make_weights(g, 1, "hard")
    px = C.synth_pixels(2, g, 4)
    rel = C.rel_l2(C.forward_hf(C.build_hf_model(flat, g), px), C.forward_np(flat, px, g))
    print(f"vit hard, 12 layers: HF fp32 vs fp64 oracle rel-L2 {rel.max():.2e}")
    assert rel.max() < 2e-5
    for eos in (2, T.EOS):
        tgeo = T.geometry(layers=12, eos_id=eos)
        tflat = T.make_weights(tgeo, 1, "hard")
        ids, lens = text_batch()
        keep = [0, 2, 3, 4]  # HF pools over the whole padded row: a 1-token item or one without <|endoftext|> pools padding
        ids, lens = ids[keep, :77], lens[keep]
        rel = T.rel_l2(T.forward_hf(T.build_hf_model(tflat, tgeo), ids, lens), T.forward_np(tflat, ids, lens, tgeo))
        print(f"text hard eos {eos}, 12 layers: HF fp32 vs fp64 oracle rel-L2 {rel.max():.2e}")
        assert rel.max() < 2e-5


def test_oracle_matches_the_hard_goldens():
    gv = np.load(os.path.join(ROOT, "tests", "golden", "clip_hard_golden.npz"))
    for case, (layers, wseed, n, pseed) in vg.CASES.items():
        g, flat, px = vg.case_inputs(case)
        assert bytes(gv[f"{case}_digest"]) == hashlib.sha256(C.pack_blob(flat, g).tobytes()).digest()
        assert float(px.astype(np.float64).sum()) == float(gv[f"{case}_px_sum"][0])
        rel = C.rel_l2(C.forward_np(flat, px, g), gv[f"{case}_emb"])
        print(f"{case}: fp64 oracle vs HF fp32 golden rel-L2 {rel.max():.2e}")
        assert rel.max() < 2e-5
    gt = np.load(os.path.join(ROOT, "tests", "golden", "clip_text_hard_golden.npz"))
    for case in tg.CASES:
        g, flat, ids, lens = tg.case_inputs(case)
        assert bytes(gt[f"{case}_digest"]) == hashlib.sha256(T.pack_blob(flat, g).tobytes()).digest()
        assert np.array_equal(gt[f"{case}_ids"], ids) and np.array_equal(gt[f"{case}_lens"], lens)
        rel = T.rel_l2(T.forward_np(flat, ids, lens, g), gt[f"{case}_emb"])
        print(f"{case}: fp64 oracle vs HF fp32 golden rel-L2 {rel.max():.2e}")
        assert rel.max() < 2e-5


def test_hard_parity_floor():
    """The emulated fp16-operand floor the hard bars rest on: the chain emulations at 12 layers against the fp64 oracle, on
    the 12-layer golden cases."""
    for case in [c for c in vg.CASES if vg.CASES[c][0] == 12]:
        g, flat, px = vg.case_inputs(case)
        out = emulate_vit_chain(FC.VitChain(flat, g, px, KE.fold_ln32), keep=False)[-1]["out"]
        rel = C.rel_l2(out, C.forward_np(flat, px, g)).max()
        print(f"vit {case}: emulated floor {rel:.2e} (bar {HARD_BAR_VIT:g})")
        assert rel < HARD_BAR_VIT / 2
    for case in [c for c in tg.CASES if tg.CASES[c][0] == 12]:
        g, flat, ids, lens = tg.case_inputs(case)
        out = emulate_clip_text_chain(CT.ClipTextChain(flat, g, ids, lens, KE.fold_ln32), keep=False)[-1]["out"]
        rel = T.rel_l2(out, T.forward_np(flat, ids, lens, g)).max()
        print(f"text {case}: emulated floor {rel:.2e} (bar {HARD_BAR_TEXT:g})")
        assert rel < HARD_BAR_TEXT / 2


# ================================================================================================ GPU

_T0 = time.perf_counter()


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()
    print(f"\ntest_gpu_pre_ln_chain: {time.perf_counter() - _T0:.1f} s wall time")


@gpu
def test_vit_chain_hard(rt):
    ch = vit_case("hard", fold=FC.gpu_fold(rt))
    model = rt.ImageEmbedModel(C.geometry_dict(ch.g), C.pack_blob(ch.flat, ch.g))
    margins = {}
    last = FC.run_chain("vit hard", ch, lambda k: model.debug_trace(ch.pixels, k), margins)
    FC.print_margins("vit hard", margins)
    assert last["n_total"] == 5 * ch.g.layers + 4 and max(margins.values()) < 1
    assert np.array_equal(model.embed(ch.pixels).view(np.uint32), last["out"].view(np.uint32)), "embed() differs from the trace"
    print(f"vit hard: rel-L2 against the fp64 oracle {C.rel_l2(last['out'], oracle(ch)).max():.3e}")


@gpu
@pytest.mark.parametrize("eos_id", [2, T.EOS])
def test_clip_text_chain_hard(rt, eos_id):
    ch = text_case("hard", eos_id, fold=FC.gpu_fold(rt))
    model = rt.ClipTextModel(ch.g, T.pack_blob(ch.flat, ch.g))
    margins = {}
    last = FC.run_chain(f"clip_text hard eos {eos_id}", ch, lambda k: model.debug_trace(ch.ids, ch.lens, k), margins)
    FC.print_margins(f"clip_text hard eos {eos_id}", margins)
    assert last["n_total"] == 5 * ch.g["layers"] + 2 and max(margins.values()) < 1
    e = model.embed(ch.ids[:, :77], ch.lens)
    assert np.array_equal(e.view(np.uint32), last["out"].view(np.uint32)), "embed() differs from the traced pooled output"
    print(f"clip_text hard eos {eos_id}: rel-L2 against the fp64 oracle {T.rel_l2(last['out'], oracle(ch)).max():.3e}")


@gpu
def test_vit_full_wave_chain_hard(rt):
    t0 = time.perf_counter()
    g = C.VitGeometry(layers=2)
    flat = C.make_weights(g, 1, "hard")
    model = rt.ImageEmbedModel(C.geometry_dict(g), C.pack_blob(flat, g))
    B, S = FW.wave_shapes(rt.wave_capacity_items() * 512)["vit"]
    px = C.synth_pixels(B, g, 4)
    ch = FC.VitChain(flat, g, px, FC.gpu_fold(rt), rows=FW.sample_rows(B, S))
    print(f"\nvit hard: {FW.coverage(ch.rows, B, S)}")
    last = FW._run("vit hard", ch, lambda k: model.debug_trace(px, k), rt.wave_capacity_items() * 512, t0)
    assert last["n_total"] == 5 * g.layers + 4
    assert np.array_equal(model.embed(px).view(np.uint32), last["out"].view(np.uint32)), "embed() differs from the trace"


@gpu
def test_clip_text_full_wave_chain_hard(rt):
    t0 = time.perf_counter()
    S, max_len = 128, 77
    g = T.geometry(layers=2, eos_id=T.EOS)
    flat = T.make_weights(g, 1, "hard")
    model = rt.ClipTextModel(g, T.pack_blob(flat, g))
    cap = model.debug_cap_rows()
    B = cap // S
    lens = FW.ragged_lens(B, S, seed=S, max_len=max_len)
    ids = T.synth_ids(lens, S, seed=5)
    ch = CT.ClipTextChain(flat, g, ids, lens, FC.gpu_fold(rt), rows=FW.sample_rows(B, S))
    print(f"\nclip_text hard: {FW.coverage(ch.rows, B, S)}")
    last = FW._run("clip_text hard", ch, lambda k: model.debug_trace(ids, lens, k), cap, t0)
    assert last["n_total"] == 5 * g["layers"] + 2
    assert np.array_equal(model.embed(ids[:, :max_len], lens).view(np.uint32), last["out"].view(np.uint32)), "embed() differs"


@gpu
@pytest.mark.parametrize("case", list(vg.CASES))
def test_vit_hard_golden_parity(rt, case):
    gv = np.load(os.path.join(ROOT, "tests", "golden", "clip_hard_golden.npz"))
    g, flat, px = vg.case_inputs(case)
    model = rt.ImageEmbedModel(C.geometry_dict(g), C.pack_blob(flat, g))
    emb = model.embed(px)
    rel = C.rel_l2(emb, gv[f"{case}_emb"])
    print(f"vit hard {case}: rel-L2 vs HF fp32 {rel.max():.3e} (bar {HARD_BAR_VIT:g})")
    assert np.allclose(np.linalg.norm(emb, axis=1), 1, atol=1e-5) and rel.max() <= HARD_BAR_VIT, rel


@gpu
@pytest.mark.parametrize("case", list(tg.CASES))
def test_clip_text_hard_golden_parity(rt, case):
    gt = np.load(os.path.join(ROOT, "tests", "golden", "clip_text_hard_golden.npz"))
    g, flat, ids, lens = tg.case_inputs(case)
    model = rt.ClipTextModel(g, T.pack_blob(flat, g))
    emb = model.embed(gt[f"{case}_ids"], gt[f"{case}_lens"])
    rel = T.rel_l2(emb, gt[f"{case}_emb"])
    print(f"clip_text hard {case}: rel-L2 vs HF fp32 {rel.max():.3e} (bar {HARD_BAR_TEXT:g})")
    assert np.allclose(np.linalg.norm(emb, axis=1), 1, atol=1e-5) and rel.max() <= HARD_BAR_TEXT, rel
