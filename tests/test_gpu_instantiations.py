"""Conformance by instantiation: every kernel template instantiation a launcher can select, checked against its fp64
reference at the shapes where tiled kernels go wrong, one parametrised test per instantiation.

tests/instantiations.py restates each launcher's selection rule and indexes the reachable instantiations.  Without a GPU:

  * the kernels compiled into libb200rt.so (cuobjdump, demangled) are exactly the reachable set -- a compiled instantiation
    nothing selects fails, and so does a selectable one that is not compiled;
  * the Python rules agree with the launch contract kernels.h documents, over every (epi, N mod 256, parts_in, stats_in)
    combination, and every production launch and debug operand selects the instantiation the index lists for it;
  * the per-model edge-case parametrisations (test_gpu_gemm_cluster.EPILOGUES, the GEMM_CASES of bge-small and bge-large,
    the CLIP text tower's 4-partial cases) jointly reach every launch_gemm instantiation, and this file's attention and row
    parametrisations reach every attention and row-kernel instantiation.

On the GPU, for each instantiation: GEMMs at M = 1, 129 (the partner tile past M) and 8320, K with fewer k-blocks than ring
stages where the geometry allows it, one cluster walking every pair (sms = 2) bitwise equal to 7, 131 and every SM, the
LayerNorm path on and off where both select the instantiation, and the residual epilogue's emitted partials; attention with
lengths on every 64-key boundary at S = 512 and an odd S, one valid key (exactly V[0]), Q = 0 (the mean of the valid values)
and launch widths on both sides of the query-tile split; the row kernels at every width with n_items not a multiple of 8 and
S = 1.  Each test prints the worst err/tol of its instantiation (< 1 passes)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import attention_refs as AR
import clip_text_refs as CT
import instantiations as IX
import kernel_refs as KR
import mean_pool_refs as MP
import rerank_refs as RR
import test_gpu_gemm_cluster as GC
from test_gpu_kernels import _gemm_case

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint16 if x.dtype == np.float16 else np.uint32)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


# ================================================================================================ CPU: the index is the library

def _tool(name):
    found = shutil.which(name)
    if found:
        return found
    for root in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if root and os.path.exists(os.path.join(root, "bin", name)):
            return os.path.join(root, "bin", name)
    pytest.fail(f"{name} (CUDA toolkit) not found: cannot list the library's kernels")


def _arg(a):
    m = re.fullmatch(r"\((int|bool)\)(-?\d+)", a.strip())
    assert m, a
    return bool(int(m.group(2))) if m.group(1) == "bool" else int(m.group(2))


def _key(demangled):
    """'void b200::gemm::gemm_kernel<(int)0, (int)256, (int)6>(...)' -> ('gemm_kernel', 0, 256, 6)."""
    m = re.match(r"(?:void )?b200::\w+::(\w+)(?:<([^<>]*)>)?\(", demangled)
    assert m, demangled
    return (m.group(1),) + (tuple(_arg(a) for a in m.group(2).split(",")) if m.group(2) else ())


def compiled_kernels(lib):
    """The instantiation key of every kernel in the library's sm_90a code."""
    res = subprocess.run([_tool("cuobjdump"), "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    mangled = re.findall(r"Function (\S+):", res)
    assert mangled, "no kernels found in " + lib
    demangled = subprocess.run([_tool("cu++filt")], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout
    return [_key(d) for d in demangled.split("\n") if d.strip()]


def test_compiled_kernels_are_the_reachable_instantiations():
    import b200rt

    assert os.path.exists(b200rt.LIB_PATH), "libb200rt.so is not built"
    got = compiled_kernels(b200rt.LIB_PATH)
    assert len(got) == len(set(got))
    unreachable = sorted(set(got) - set(IX.REACHABLE), key=str)
    missing = sorted(set(IX.REACHABLE) - set(got), key=str)
    print(f"{len(got)} kernels compiled, {len(IX.REACHABLE)} reachable "
          f"({sum(k[0] == IX.GEMM for k in got)} GEMM, {sum(k[0] == IX.ATTN for k in got)} attention)")
    assert not unreachable, f"compiled but no launcher selects them: {[IX.describe(k) for k in unreachable]}"
    assert not missing, f"selectable but not compiled: {[IX.describe(k) for k in missing]}"


# ================================================================================================ CPU: the rules are kernels.h's

def _documented_gemm(epi, N, K, stats_in, parts_in):
    """launch_gemm as kernels.h documents it: N % 128 == 0, K % 64 == 0; with stats_in, parts_in is the LayerNorm'd width
    (K for epi 0/1/3, N for epi 2) / 128, that width 768 or 384, 1024 for epi 0/1/2 with N % 256 == 0, or 512 for epi 0/3
    with N % 256 == 0.  Tiles are 256 wide when N % 256 == 0, else 128; without stats_in the 6-partial instantiation runs."""
    if epi not in (0, 1, 2, 3) or N < 128 or K < 64 or N % 128 or K % 64:
        return None
    if stats_in:
        width = N if epi == 2 else K
        if parts_in * 128 != width:
            return None
        wide = N % 256 == 0
        if not (width in (768, 384) or (width == 1024 and epi in (0, 1, 2) and wide) or (width == 512 and epi in (0, 3) and wide)):
            return None
    return (IX.GEMM, epi, 256 if N % 256 == 0 else 128, parts_in if stats_in else 6)


N_WALK = (128, 256, 384, 512, 640, 768, 1024, 1152, 1536, 2048, 2304, 3072, 4096, 6144, 100)
K_WALK = (64, 128, 192, 384, 512, 640, 768, 1024, 1536, 2048, 3072, 4096, 96)


def test_gemm_rule_matches_the_documented_contract():
    """Every (epi, N, K, stats_in NULL or not, parts_in) over N of both residues mod 256: launch_gemm's selection (or refusal)
    is the one kernels.h documents."""
    n = 0
    for epi in range(-1, 5):
        for N in N_WALK:
            for K in K_WALK:
                for stats in (False, True):
                    for parts in (range(0, 10) if stats else (6,)):
                        want = _documented_gemm(epi, N, K, stats, parts)
                        got = IX.gemm(epi, N, K, stats, parts)
                        assert got == want, (epi, N, K, stats, parts, got, want)
                        n += 1
    print(f"{n} launch_gemm operand sets agree with kernels.h")


def test_fused_epilogue_and_attention_rules_match_the_documented_contract():
    for N in N_WALK:
        for K in K_WALK:
            for stats in (False, True):
                for parts in range(0, 10):
                    # SPLADE: stats_in required, the LayerNorm of A K wide (768, 384 or 1024); N % 256 == 0
                    want = (IX.GEMM, 4, 256, parts) if stats and N % 256 == 0 and K in (768, 384, 1024) and parts * 128 == K else None
                    assert IX.gemm_splade(N, K, stats, parts) == want, (N, K, stats, parts)
                    # rotary / SwiGLU: K = 768 (6 partials, or no LayerNorm), N % 256 == 0
                    ok = N % 256 == 0 and K == 768 and (not stats or parts == 6)
                    assert IX.gemm_rope(N, K, stats, parts) == ((IX.GEMM, 5, 256, 6) if ok else None)
                    assert IX.gemm_swiglu(N, K, stats, parts) == ((IX.GEMM, 6, 256, 6) if ok else None)
    for d in (16, 32, 48, 64, 128):
        for nh in (8, 12, 16, 20):
            for causal in (False, True):
                ok = (d, nh) == (64, 8) if causal else (d, nh) in ((64, 12), (32, 12), (64, 16))
                assert IX.attention(d, nh, causal) == ((IX.ATTN, d, nh, causal) if ok else None)
    for W in (256, 384, 512, 768, 1024, 1536):
        for segs in (False, True):
            ok = W in (768, 384, 1024) or (W == 512 and not segs)
            assert IX.embed(W, segs) == (("embed_kernel", W, segs) if ok else None)
        for name in ("pool_normalize", "mean_pool_normalize", "cls_head", "mlm_ln_stats"):
            assert IX.ROW_RULES[name](W) == ((f"{name}_kernel", W) if W in (768, 384, 1024) else None)


def test_gemm_refusals_are_the_documented_ones():
    """Spot checks of the C++ refusals kernels.h spells out: no 8-partial quick-GELU, no 4-partial GELU or residual, no
    512- or 1024-wide LayerNorm on a 128-column tile, and no 3-partial residual on a 256-column tile (N = 384 is the only
    3-partial residual width)."""
    assert IX.gemm(3, 1024, 1024, True, 8) is None
    assert IX.gemm(1, 2048, 512, True, 4) is None and IX.gemm(2, 512, 512, True, 4) is None
    assert IX.gemm(0, 1152, 1024, True, 8) is None and IX.gemm(0, 384, 512, True, 4) is None
    assert all(IX.gemm(2, N, K, True, 3) in (None, (IX.GEMM, 2, 128, 3)) for N in N_WALK for K in K_WALK)


def test_every_listed_launch_selects_its_instantiation():
    """Each production launch and each debug-entry operand set in the index maps through the rules to the instantiation it is
    listed under; every reachable instantiation has at least one of them."""
    for model, launch, key in IX.production_launches():
        assert key in IX.REACHABLE, (model, launch, key)
    for key, entry in IX.REACHABLE.items():
        assert entry["production"] or entry["debug"], key
        op = entry["debug"]
        if op is None:
            continue
        e = op["entry"]
        if e == "debug_gemm":
            assert IX.gemm(op["epi"], op["N"], op["K"], op["ln"] is not None, op["ln"] or 6) == key, (key, op)
        elif e == "debug_gemm_splade":
            assert IX.gemm_splade(512, op["K"], True, op["K"] // 128) == key
        elif e == "debug_gemm_rope":
            assert IX.gemm_rope(op["N"], 768, True) == key
        elif e == "debug_gemm_swiglu":
            assert IX.gemm_swiglu(op["N"], 768, True) == key
        elif e == "debug_attention":
            assert IX.attention(op["head_dim"], op["heads"], op["causal"]) == key
        elif e == "debug_embed":
            assert IX.embed(op["hidden"], False) == key
        elif e == "debug_embed_segs":
            assert IX.embed(op["hidden"], True) == key
        elif e in ("debug_pool_normalize", "debug_mean_pool_normalize", "debug_cls_head", "debug_mlm_ln_stats"):
            assert IX.ROW_RULES[e[len("debug_"):]](op["hidden"]) == key
        else:
            assert e in ("debug_attention_stream", "debug_clip_text_pool") or key[0] in IX.PLAIN_KERNELS, (key, op)
    print("\n".join(IX.table_lines()))


def _existing_gemm_cases():
    """(source, launch_gemm key) of the per-model GEMM edge-case parametrisations, each mapped through the rule as its test
    builds the operands: _gemm_case in test_gpu_gemm_cluster, test_gpu_bge_small and test_gpu_bge_large folds (epi 0/1/3) or
    re-applies (epi 2) a LayerNorm of the K- (N-) wide rows."""
    import test_gpu_bge_large as BL
    import test_gpu_bge_small as BS
    import test_gpu_clip_text as CTT

    def ln_on(src, epi, N, K):
        return src, IX.gemm(epi, N, K, True, (N if epi == 2 else K) // 128)

    out = [ln_on("test_gpu_gemm_cluster.EPILOGUES", e, N, K) for e, N, K, _ in GC.EPILOGUES]
    out += [ln_on("test_gpu_bge_small.GEMM_CASES", e, N, K) for e, N, K in BS.GEMM_CASES]
    out += [ln_on("test_gpu_bge_large.GEMM_CASES", e, N, K) for e, N, K in BL.GEMM_CASES]
    out += [("test_gpu_clip_text.LN512_CASES", IX.gemm(e, N, 512, True, 4)) for e, N in CTT.LN512_CASES]
    # the residual epilogue without stats_in at N = 384 (test_residual_epilogue_three_partials_without_stats_in)
    out += [("test_gpu_bge_small.RESIDUAL_NO_LN_KS", IX.gemm(2, 384, K, False)) for K in BS.RESIDUAL_NO_LN_KS]
    out += [("test_gpu_gemm_cluster.SPLADE_KS", IX.gemm_splade(512, K, True, K // 128)) for K in GC.SPLADE_KS]
    out += [("test_gpu_gemm_cluster.ROPE_PAST_M", IX.gemm_rope(2304, 768, ln)) for _ in GC.ROPE_PAST_M for ln in (True, False)]
    out += [("test_gpu_gemm_cluster swiglu", IX.gemm_swiglu(6144, 768, True))]
    return out


def test_existing_parametrisations_reach_every_instantiation():
    """Every GEMM instantiation is reached by a per-model edge-case parametrisation, and every attention and row-kernel
    instantiation with a debug entry by this file's parametrisations: an instantiation added without a conformance case
    fails here."""
    cases = _existing_gemm_cases()
    assert all(k is not None for _, k in cases), [c for c in cases if c[1] is None]
    by_key = {}
    for src, k in cases:
        by_key.setdefault(k, set()).add(src)
    gemm_keys = {k for k in IX.REACHABLE if k[0] == IX.GEMM}
    missing = sorted(gemm_keys - set(by_key), key=str)
    for k in sorted(gemm_keys, key=str):
        print(f"{IX.describe(k)}: {', '.join(sorted(by_key.get(k, ()))) or 'NOT REACHED'}")
    assert not missing, f"no edge-case parametrisation reaches {[IX.describe(k) for k in missing]}"
    attn = {IX.attention(*c) for c in ATTENTION_CASES} | {IX.attention_stream(512)}
    assert attn == {k for k in IX.REACHABLE if k[0] in (IX.ATTN, IX.ATTN_STREAM)}, attn
    rows = {IX.ROW_RULES[name](W) if name != "embed" else IX.embed(W, segs) for name, W, segs in ROW_CASES}
    assert rows == {k for k in IX.REACHABLE if k[0] in {f"{n}_kernel" for n in IX.ROW_RULES}}, rows


# ================================================================================================ GPU: GEMM

M_EDGES = (1, 129, 8320)  # one m-tile; two, the partner tile past M; 65, an odd count over many pairs
SMS = (7, 131, 0)          # each bitwise equal to one cluster (sms = 2)
SHORT_K = 192              # 3 k-blocks: fewer than the 4 ring stages


def _gemm_variants():
    """(key, ln, N, Ks) for each launch_gemm instantiation: its debug operands with the LayerNorm on (when it has one) and off
    (when no LayerNorm still selects it, i.e. PARTS = 6); the short K where the LayerNorm does not fix K (off, or epi 2,
    whose LayerNorm is N wide)."""
    out = []
    for key in sorted((k for k in IX.REACHABLE if k[0] == IX.GEMM and k[1] <= 3), key=str):
        op = IX.REACHABLE[key]["debug"]
        epi, N, K, parts = op["epi"], op["N"], op["K"], op["ln"]
        for ln in (True, False):
            if ln and parts is None:
                continue
            if IX.gemm(epi, N, K, ln, parts or 6) != key:
                continue
            ks = [K]
            if (epi == 2 or not ln) and IX.gemm(epi, N, SHORT_K, ln, parts or 6) == key:
                ks.append(SHORT_K)
            out.append(pytest.param(key, ln, N, tuple(ks), id=f"{IX.describe(key)}-{'ln' if ln else 'no_ln'}"))
    return out


@gpu
@pytest.mark.parametrize("key,ln,N,Ks", _gemm_variants())
def test_gemm_instantiation(rt, key, ln, N, Ks):
    epi, parts = key[1], key[3]
    worst = 0.0
    for K in Ks:
        for M in (M_EDGES if K == Ks[0] else (129,)):
            args, kw = _gemm_case(epi, M, N, K, seed=M + 7 * epi + N + K + ln, ln=ln)
            want = epi == 2
            tag = f"{IX.describe(key)} ln={ln} M={M} N={N} K={K}"
            r = rt.debug_gemm(epi, *args, want_stats=want, sms=2, want_ctas=True, ln512=parts == 4 and ln, **kw)
            assert r[-1] == 2, r[-1]
            worst = max(worst, KR.check_gemm(f"{tag} sms 2", r[0], epi, *args, **kw))
            if want:
                worst = max(worst, KR.check_gemm_stats(f"{tag} sms 2: stats_out", r[2], args, **kw))
            for sms in SMS:
                g = rt.debug_gemm(epi, *args, want_stats=want, sms=sms, want_ctas=True, ln512=parts == 4 and ln, **kw)
                same = _same(g[0], r[0]) and (not want or _same(g[2], r[2]))
                assert same, f"{tag}: sms {sms} ({g[-1]} CTAs) differs bitwise from one cluster"
    print(f"{IX.describe(key)} ln={ln}: worst err/tol {worst:.3f} over M {M_EDGES}, K {Ks}; sms {SMS} bitwise equal to sms 2")


def _fused_cases(key):
    """(tag, run, check) of the SPLADE / rotary / SwiGLU instantiation at the M edges, from test_gpu_gemm_cluster's builders."""
    epi = key[1]
    out = []
    if epi == IX.EPI_SPLADE_MAX:
        K = key[3] * 128
        for B in (1, 3, 130):  # M = 64, 192 (the partner tile past M), 8320
            out.append((f"splade K={K} B={B} S=64", *GC._splade_case(B, 64, K, 2000, seed=B + K)))
    elif epi == IX.EPI_ROPE_F16:
        for B in (1, 3, 130):
            for ln in (True, False):
                out.append((f"rope M={64 * B} ln={ln}", *GC._rope_case(64 * B, 64, ln, seed=B + ln)))
    else:
        for M in M_EDGES:
            for ln in (True, False):
                out.append((f"swiglu M={M} ln={ln}", *GC._swiglu_case(M, ln, seed=M + ln)))
    return out


@gpu
@pytest.mark.parametrize("key", sorted((k for k in IX.REACHABLE if k[0] == IX.GEMM and k[1] > 3), key=str), ids=IX.describe)
def test_fused_gemm_instantiation(rt, key):
    worst = 0.0
    for tag, run, check in _fused_cases(key):
        one, ctas = run(rt, 2)
        assert ctas == 2, ctas
        worst = max(worst, check(f"{tag} sms 2", one))
        for sms in SMS:
            got, c = run(rt, sms)
            assert _same(got, one), f"{tag}: sms {sms} ({c} CTAs) differs bitwise from one cluster"
    print(f"{IX.describe(key)}: worst err/tol {worst:.3f}; sms {SMS} bitwise equal to sms 2")


# ================================================================================================ GPU: attention

ATTENTION_CASES = [(64, 12, False), (32, 12, False), (64, 16, False), (64, 8, True)]  # (head_dim, heads, causal)
ATTN_KEYS = [IX.attention(*c) for c in ATTENTION_CASES] + [IX.attention_stream(512)]
BOUNDARY_LENS = [1] + [b + d for b in range(64, 513, 64) for d in (-1, 0, 1) if b + d <= 512]


def _geom(key):
    return (64, 12, False) if key[0] == IX.ATTN_STREAM else key[1:]


def _attend(rt, key, qkv, lens, B, S, sms=0):
    lens = np.asarray(lens, np.int32)
    if key[0] == IX.ATTN_STREAM:
        return rt.debug_attention_stream(qkv, lens, B, S, sms=sms)[0]
    d, nh, causal = key[1:]
    return rt.debug_attention(qkv, lens, B, S, sms=sms, head_dim=d, heads=nh, causal=causal)[0]


def _attn_ref(key, qkv, lens, B, S):
    d, nh, causal = _geom(key)
    if causal:
        return CT.causal_attention_ref(qkv, lens, B, S, heads=nh, hd=d)
    return AR.attention_ref(qkv, lens, B, S, heads=nh, head_dim=d)


def _check_attn(tag, key, ctx, qkv, lens, B, S):
    ref, tol = _attn_ref(key, qkv, lens, B, S)
    got = np.asarray(ctx, np.float16).astype(np.float64)
    assert np.isfinite(got).all(), f"{tag}: non-finite output"
    return KR.check(tag, got, ref, tol)


def _qkv(rng, key, B, S, scale=2.0):
    d, nh, _ = _geom(key)
    return (rng.standard_normal((B * S, 3 * d * nh)) * scale).astype(np.float16)


@gpu
@pytest.mark.parametrize("key", ATTN_KEYS, ids=IX.describe)
def test_attention_lens_on_every_64_key_boundary(rt, key):
    """Lengths 1 and b - 1, b, b + 1 for every multiple b of 64 up to 512, at S = 512 and at an odd S (449; the streaming
    kernel takes S % 64 == 0 only: 576), lengths past S clamped."""
    worst = 0.0
    for S in (512, 576 if key[0] == IX.ATTN_STREAM else 449):
        lens = BOUNDARY_LENS
        B = len(lens)
        qkv = _qkv(np.random.default_rng(S + len(key)), key, B, S)
        ctx = _attend(rt, key, qkv, lens, B, S)
        worst = max(worst, _check_attn(f"{IX.describe(key)} S={S} boundary lens", key, ctx, qkv, lens, B, S))
    print(f"{IX.describe(key)}: lens on every 64-key boundary, worst err/tol {worst:.3f}")


@gpu
@pytest.mark.parametrize("key", ATTN_KEYS, ids=IX.describe)
def test_attention_single_key_and_zero_queries(rt, key):
    """One valid key: every query row is V[0] exactly.  Q = 0: every score is 0, so each row is the mean of the values it
    may see -- all valid keys, or (causal) keys 0 .. min(q, len - 1)."""
    d, nh, causal = _geom(key)
    H = d * nh
    B, S = 3, 192
    rng = np.random.default_rng(8 + d + nh)
    qkv = _qkv(rng, key, B, S, scale=3.0)
    ctx = _attend(rt, key, qkv, np.ones(B, np.int32), B, S)
    v0 = qkv.reshape(B, S, 3 * H)[:, :1, 2 * H:]
    assert _same(ctx.reshape(B, S, H), np.ascontiguousarray(np.broadcast_to(v0, (B, S, H)))), "len 1: not V[0] bitwise"
    lens = [S, 129, 64]
    qkv[:, :H] = 0.0
    ctx = _attend(rt, key, qkv, lens, B, S)
    v = qkv.reshape(B, S, 3 * H)[..., 2 * H:].astype(np.float64)
    mean = []
    for b, n in enumerate(lens):
        last = np.minimum(np.arange(S), n - 1) if causal else np.full(S, n - 1)
        csum = np.cumsum(v[b], 0)
        mean.append(csum[last] / (last + 1)[:, None])
    mean = np.concatenate(mean)
    ref, tol = _attn_ref(key, qkv, lens, B, S)
    assert np.allclose(ref, mean, rtol=1e-12, atol=1e-12)
    m = KR.check(f"{IX.describe(key)} Q = 0: mean of the visible values", ctx, mean, tol)
    print(f"{IX.describe(key)}: len 1 gives V[0] bitwise; Q = 0 worst err/tol {m:.3f}")


@gpu
@pytest.mark.parametrize("key", ATTN_KEYS, ids=IX.describe)
def test_attention_launch_widths_across_the_query_tile_split(rt, key):
    """B = 4: sms = B NH keeps one unit per (item, head), B NH + 1 splits units by query tile; 1 and 132 too.  Every launch
    bitwise equal to the one on every SM (the streaming kernel always walks query tiles: 1, 7, 131)."""
    d, nh, _ = _geom(key)
    B, S, lens = 4, 512, [512, 77, 300, 129]
    qkv = _qkv(np.random.default_rng(4), key, B, S)
    base = _attend(rt, key, qkv, lens, B, S)
    m = _check_attn(f"{IX.describe(key)} every SM", key, base, qkv, lens, B, S)
    if key[0] == IX.ATTN_STREAM:
        widths = (1, 7, 131)
    else:
        widths = (1, B * nh, B * nh + 1, 132)
        assert not IX.attention_split(B, S, B * nh, nh) and IX.attention_split(B, S, B * nh + 1, nh)
    for sms in widths:
        got = _attend(rt, key, qkv, lens, B, S, sms=sms)
        assert _same(got, base), f"{IX.describe(key)}: sms {sms} differs bitwise from every SM"
    print(f"{IX.describe(key)}: worst err/tol {m:.3f}; sms {widths} bitwise equal to every SM")


# ================================================================================================ GPU: row kernels

ROW_CASES = ([("embed", W, segs) for W in IX.TEXT_WIDTHS for segs in (False, True)] + [("embed", 512, False)]
             + [(name, W, False) for name in ("pool_normalize", "mean_pool_normalize", "cls_head", "mlm_ln_stats") for W in IX.TEXT_WIDTHS])
ROW_SHAPES = [(1, 13), (7, 133)]  # (S, n_items): S = 1, and items not a multiple of the 8 warps per block


def _rows(rng, n, W, mean=0.3):
    x = (rng.standard_normal((n, W)) * 1.5 + mean + np.repeat(rng.standard_normal(W // 64) * 0.5, 64)[None, :]).astype(np.float32)
    return KR.split_hilo(x)


def _ln_params(rng, W):
    return (1.0 + 0.3 * rng.standard_normal(W)).astype(np.float32), (0.2 * rng.standard_normal(W)).astype(np.float32)


def _row_case(rt, name, W, segs, S, n, rng):
    if name == "embed":
        vocab = 50
        word = (rng.standard_normal((vocab, W)) + np.repeat(rng.standard_normal(W // 128) * 3.0, 128)[None, :]).astype(np.float32)
        pos = rng.standard_normal((S, W)).astype(np.float32)
        ids = rng.integers(0, vocab, size=n * S).astype(np.int32)
        if segs:
            type2 = rng.standard_normal((2, W)).astype(np.float32)
            sg = rng.integers(-1, S + 2, size=n).astype(np.int32)
            hi, lo, st = rt.debug_embed_segs(ids, sg, word, pos, type2, S, hidden=W)
            return RR.check_embed_segs(f"embed segs W={W} S={S} n={n}", hi, lo, st, ids, sg, word, pos, type2, S)
        type0 = np.zeros(W, np.float32) if W == 512 else (0.3 * rng.standard_normal(W)).astype(np.float32)
        hi, lo, st = rt.debug_embed(ids, word, pos, type0, S, hidden=W)
        return KR.check_embed(f"embed W={W} S={S} n={n}", hi, lo, st, ids, word, pos, type0, S)
    hi, lo = _rows(rng, n * S, W)
    g, b = _ln_params(rng, W)
    if name == "pool_normalize":
        out = rt.debug_pool_normalize(hi, lo, g, b, S, 1e-12, hidden=W)
        return KR.check_pool_normalize(f"pool_normalize W={W} S={S} n={n}", out, hi, lo, g, b, S, 1e-12)
    if name == "mean_pool_normalize":
        lens = rng.integers(0, S + 2, size=n).astype(np.int32)  # 0 and S + 1 clamp to [1, S]
        out = rt.debug_mean_pool_normalize(hi, lo, g, b, lens, S, 1e-12, hidden=W)
        return MP.check_mean_pool_normalize(f"mean_pool_normalize W={W} S={S} n={n}", out, hi, lo, g, b, lens, S, 1e-12)
    if name == "cls_head":
        L = 3
        pw = (rng.standard_normal((W, W)) * 1.5 / np.sqrt(W)).astype(np.float32)
        pb = (0.1 * rng.standard_normal(W)).astype(np.float32)
        cw = (rng.standard_normal((L, W)) * 0.3).astype(np.float32)
        cb = rng.standard_normal(L).astype(np.float32)
        out = rt.debug_cls_head(hi, lo, g, b, pw, pb, cw, cb, S, 1e-12, hidden=W)
        return RR.check_cls_head(f"cls_head W={W} S={S} n={n}", out, hi, lo, g, b, pw, pb, cw, cb, S, 1e-12)
    u = (hi.astype(np.float32) * 1.3).astype(np.float16)
    st, vmax = rt.debug_mlm_ln_stats(u, n_max=4099)
    assert (vmax == 0).all(), "the max buffer was not zeroed"
    return KR.check_partials(f"mlm_ln_stats W={W} rows={n * S}", st, u.astype(np.float64))


@gpu
@pytest.mark.parametrize("name,W,segs", ROW_CASES, ids=[f"{n}-{W}{'-segs' if s else ''}" for n, W, s in ROW_CASES])
def test_row_kernel_instantiation(rt, name, W, segs):
    key = IX.embed(W, segs) if name == "embed" else IX.ROW_RULES[name](W)
    worst = 0.0
    for S, n in ROW_SHAPES:
        worst = max(worst, _row_case(rt, name, W, segs, S, n, np.random.default_rng(W + S + n + segs)))
    print(f"{IX.describe(key)}: worst err/tol {worst:.3f} at (S, n_items) {ROW_SHAPES}")
