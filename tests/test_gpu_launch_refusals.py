"""The kernel launchers are the only judge of a debug entry's operands.

A launcher refuses operands outside its contract with cudaErrorInvalidValue before it enqueues anything, and the engine
returns that refusal as B200RT_E_INVALID without poisoning the runtime.  The debug entries keep only the checks their own
host buffers need and the debug ABI's policy (the B200RT_DEBUG_GEMM_LN512 flag), so over each operand grid below a call must
be accepted exactly when tests/instantiations.py selects an instantiation for it and that policy allows it, and refused with
E_INVALID otherwise.  After each walk a valid call still succeeds: no refusal poisoned the process.

The SPLADE finalize case runs in a subprocess: a refusal there once reached the caller as a CUDA error and poisoned the
process for good."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import instantiations as IX

gpu = pytest.mark.gpu

M = 64  # GEMM rows


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


def _accepted(rt, call):
    """True when the call succeeds, False when it is refused with E_INVALID; any other error fails the test."""
    try:
        call()
        return True
    except rt.B200RTError as e:
        assert e.code == rt.E_INVALID, e
        return False


def _walk(rt, cases):
    """cases: (description, wanted acceptance, call).  Every call must meet its expectation, and a valid GEMM must still run
    afterwards."""
    wrong = [(what, want) for what, want, call in cases if _accepted(rt, call) != want]
    n_ok = sum(want for _, want, _ in cases)
    print(f"{len(cases)} calls, {n_ok} accepted as expected, {len(cases) - n_ok} refused, {len(wrong)} disagree with the rules")
    assert not wrong, wrong[:20]
    out, _ = rt.debug_gemm(0, np.ones((M, 768), np.float16), np.zeros((768, 768), np.float16), np.full(768, 0.5, np.float32))
    assert (out == 0.5).all()


def _z16(*shape):
    return np.zeros(shape, np.float16)


def _z32(*shape):
    return np.zeros(shape, np.float32)


@gpu
def test_debug_gemm_accepts_exactly_the_selectable_operands(rt):
    cases = []
    for epi in range(4):
        for N in (100, 128, 384, 512, 768, 1024, 1152):
            for K in (64, 96, 384, 512, 768, 1024):
                ln_w = N if epi == IX.EPI_BIAS_RES_SPLIT else K
                parts = ln_w // 128
                for ln in (False, True):
                    for ln512 in (False, True) if ln else (False,):
                        want = IX.gemm(epi, N, K, ln, parts) is not None and not (ln and ln_w == 512 and not ln512)
                        kw = dict(resid=_z32(M, N) if epi == IX.EPI_BIAS_RES_SPLIT else None, ln512=ln512)
                        if ln:
                            kw.update(ln_stats=_z32(M, max(parts, 1), 2), ln_gamma=np.ones(N, np.float32), ln_beta=_z32(N))
                        call = lambda epi=epi, N=N, K=K, kw=kw: rt.debug_gemm(epi, _z16(M, K), _z16(N, K), _z32(N), **kw)  # noqa: E731
                        cases.append(((epi, N, K, ln, ln512), want, call))
    _walk(rt, cases)


@gpu
def test_fused_gemms_accept_exactly_the_selectable_operands(rt):
    cases = []
    S = 64
    for N in (100, 256, 384, 512, 768):
        for K in (64, 96, 384, 512, 768, 1024):
            vocab = min(N, 100)
            want = IX.gemm_splade(N, K, True, K // 128) is not None
            call = lambda N=N, K=K, vocab=vocab: rt.debug_gemm_splade(_z16(S, K), _z16(vocab, K), _z32(N), _z32(S, K // 128, 2),  # noqa: E731
                                                                      np.array([S], np.int32), S, N, 1e-12)
            cases.append((("splade", N, K), want, call))
    table = _z32(S, 32, 2)
    for N in (100, 128, 256, 768, 2304):
        for stats in (None, _z32(M, 6, 2)):
            want = IX.gemm_rope(N, 768, stats is not None) is not None
            call = lambda N=N, stats=stats: rt.debug_gemm_rope(_z16(M, 768), _z16(N, 768), _z32(N), stats, table, S, 0, 1e-12)  # noqa: E731
            cases.append((("rope", N, stats is not None), want, call))
            want = IX.gemm_swiglu(N, 768, stats is not None) is not None
            call = lambda N=N, stats=stats: rt.debug_gemm_swiglu(_z16(M, 768), _z16(N, 768), _z32(N), stats, 1e-12)  # noqa: E731
            cases.append((("swiglu", N, stats is not None), want, call))
    _walk(rt, cases)


@gpu
def test_debug_attention_accepts_exactly_the_selectable_operands(rt):
    cases = []
    for head_dim in (32, 48, 64):
        for heads in (8, 12, 16):
            for causal in (False, True):
                for S in (64, 512, 576):
                    want = IX.attention(head_dim, heads, causal) is not None and S <= IX.ATTN_MAX_S
                    call = lambda hd=head_dim, nh=heads, c=causal, S=S: rt.debug_attention(  # noqa: E731
                        _z16(S, 3 * hd * nh), np.array([S], np.int32), 1, S, head_dim=hd, heads=nh, causal=c)
                    cases.append(((head_dim, heads, causal, S), want, call))
    for S in (32, 64, 96, 8192, 8256):
        want = IX.attention_stream(S) is not None
        call = lambda S=S: rt.debug_attention_stream(_z16(S, 2304), np.array([S], np.int32), 1, S)  # noqa: E731
        cases.append((("stream", S), want, call))
    _walk(rt, cases)


@gpu
def test_row_entries_accept_exactly_the_selectable_widths(rt):
    n, S = 3, 4
    cases = []
    for W in (256, 384, 512, 768, 1024):
        ids = np.zeros(n * S, np.int32)
        hi = _z16(n * S, W)
        g, b = np.ones(W, np.float32), _z32(W)
        calls = {
            "embed": (IX.embed(W, False), lambda W=W: rt.debug_embed(ids, _z32(5, W), _z32(S, W), _z32(W), S, hidden=W)),
            "embed_segs": (IX.embed(W, True), lambda W=W: rt.debug_embed_segs(ids, np.full(n, 2, np.int32), _z32(5, W), _z32(S, W),
                                                                              _z32(2, W), S, hidden=W)),
            "pool_normalize": (IX.pool_normalize(W), lambda W=W, hi=hi, g=g, b=b: rt.debug_pool_normalize(hi, hi, g, b, S, 1e-12, hidden=W)),
            "mean_pool_normalize": (IX.mean_pool_normalize(W), lambda W=W, hi=hi, g=g, b=b: rt.debug_mean_pool_normalize(
                hi, hi, g, b, np.full(n, S, np.int32), S, 1e-12, hidden=W)),
            "cls_head": (IX.cls_head(W), lambda W=W, hi=hi, g=g, b=b: rt.debug_cls_head(hi, hi, g, b, _z32(W, W), _z32(W), _z32(2, W), _z32(2),
                                                                                      S, 1e-12, hidden=W)),
            "mlm_ln_stats": (IX.mlm_ln_stats(W), lambda hi=hi: rt.debug_mlm_ln_stats(hi, n_max=8)),
        }
        for name, (key, call) in calls.items():
            cases.append(((name, W), key is not None, call))
    _walk(rt, cases)


@gpu
def test_splade_finalize_refusal_leaves_the_runtime_usable():
    """n_items = 65536 is past the launch grid's y limit: the launcher refuses it, and the process stays usable."""
    code = textwrap.dedent("""
        import numpy as np
        import b200rt

        b200rt.init(devices=[0])
        try:
            b200rt.debug_splade_finalize(np.zeros((65536, 256), np.uint32), 1)
            print("accepted")
        except b200rt.B200RTError as e:
            print("refused", e.code)
        try:
            out = b200rt.debug_splade_finalize(np.zeros((2, 256), np.uint32), 1)
            print("valid call", out.shape, float(out.max()))
        except b200rt.B200RTError as e:
            print("valid call failed", e.code)
        b200rt.shutdown()
    """)
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "modal-examples_b200")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([pkg] + [p for p in os.environ.get("PYTHONPATH", "").split(os.pathsep) if p]))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    import b200rt

    assert f"refused {b200rt.E_INVALID}" in r.stdout, r.stdout
    assert "valid call (2, 1) 0.0" in r.stdout, r.stdout
