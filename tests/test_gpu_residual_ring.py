"""The residual GEMM epilogue (EPI_BIAS_RES_SPLIT) reads its tile's residual y = hi + lo through the GEMM's operand ring: after a
tile's last k-block the producer takes BN / 64 more ring entries, one per 64-column chunk, each a TMA of the chunk's hi box
[128 x 64] and lo box into one stage (gemm_sm90.cu, the protocol comment at the top).

Without a GPU: the producer's and the consumers' walks through the ring, restated from the kernel, give both ranks of a
cluster the same (stage, phase, operand-or-residual) sequence, and every entry's expect_tx equals the bytes its TMA loads
deliver to that CTA -- at per-tile entry counts that are not a multiple of the four stages (K = 64, 192, 768, 3072 with
BN = 256 and 128), over several tiles per cluster.

On the GPU: b200rt.debug_gemm epi 2 over K in {64, 192, 768, 3072}, N in {384, 768, 1024}, M in {1, 127, 129, 257, 1000},
with and without the LayerNorm re-applied, against the fp64 reference (output and emitted partials), and bitwise equal at
sms = 1, 2, 3 and every SM -- one cluster then walks many ring laps with residual entries interleaved."""
import os
import re

import numpy as np
import pytest

import kernel_refs as KR
from test_gpu_kernels import _gemm_case

gpu = pytest.mark.gpu

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "modal-examples_b200", "csrc", "gemm_sm90.cu")

BM, BK, STAGES, CM = 128, 64, 4, 2
A_BYTES = BM * BK * 2
W_BOX_BYTES = 128 * BK * 2
RES_BOX_BYTES = BM * 64 * 2


def test_ring_constants_are_the_kernels():
    src = open(SRC).read()
    for name, value in (("BM", BM), ("STAGES", STAGES), ("CM", CM)):
        assert re.search(rf"\b{name} = {value}\b", src), name
    assert re.search(r"\bBK = 64\b", src)
    assert re.search(r"RES_BOX_BYTES = BM \* 64 \* 2;", src)


# ================================================================================================ CPU: the ring walk

def _slots(M, N, BN, clusters, rank):
    """(m0, n0) of the tiles rank `rank` of every cluster walks, cluster by cluster: slot t = CM p + r, t += CM clusters."""
    num_n = N // BN
    num_slots = -(-M // (CM * BM)) * num_n * CM
    walks = []
    for c in range(clusters):
        tiles = []
        for t in range(CM * c + rank, num_slots, CM * clusters):
            p = t // CM
            tiles.append((((p // num_n) * CM + t % CM) * BM, (p % num_n) * BN))
        walks.append(tiles)
    return walks


def producer_walk(M, N, K, BN, clusters, rank):
    """Per cluster, the producer of `rank`: (stage, phase, kind, expect_tx, {smem offset: (bytes, loader rank, what)}) for
    every entry, in order.  W box b of an operand entry is loaded by rank b % CM and multicast into both CTAs."""
    out = []
    for tiles in _slots(M, N, BN, clusters, rank):
        stage, phase, seq = 0, 0, []
        for m0, n0 in tiles:
            for kb in range(K // BK):
                loads = {0: (A_BYTES, rank, ("A", kb * BK, m0))}
                for b in range(BN // 128):
                    loads[A_BYTES + b * W_BOX_BYTES] = (W_BOX_BYTES, b % CM, ("W", kb * BK, n0 + 128 * b))
                seq.append((stage, phase, "operand", A_BYTES + BN * BK * 2, loads))
                stage, phase = (0, phase ^ 1) if stage + 1 == STAGES else (stage + 1, phase)
            for q in range(BN // 64):
                loads = {0: (RES_BOX_BYTES, rank, ("hi", n0 + 64 * q, m0)), RES_BOX_BYTES: (RES_BOX_BYTES, rank, ("lo", n0 + 64 * q, m0))}
                seq.append((stage, phase, "residual", 2 * RES_BOX_BYTES, loads))
                stage, phase = (0, phase ^ 1) if stage + 1 == STAGES else (stage + 1, phase)
        out.append(seq)
    return out


def consumer_walk(M, N, K, BN, clusters, rank):
    """Per cluster, the consumers of `rank`: (stage, phase, kind) of every full[stage] wait, in order -- the k-block loop,
    then one wait per 64-column chunk of the epilogue."""
    out = []
    for tiles in _slots(M, N, BN, clusters, rank):
        stage, phase, seq = 0, 0, []
        for _ in tiles:
            for kind, n in (("operand", K // BK), ("residual", BN // 64)):
                for _ in range(n):
                    seq.append((stage, phase, kind))
                    stage, phase = (0, phase ^ 1) if stage + 1 == STAGES else (stage + 1, phase)
        out.append(seq)
    return out


RING_CASES = [(K, BN) for K in (64, 192, 768, 3072) for BN in (256, 128)]


def test_ring_cases_cover_entry_counts_off_the_stage_count():
    counts = {K // BK + BN // 64 for K, BN in RING_CASES}
    assert any(n % STAGES for n in counts), counts


@pytest.mark.parametrize("K,BN", RING_CASES)
def test_ring_walk_lockstep_and_byte_counts(K, BN):
    entries = K // BK + BN // 64
    N = 3 * BN
    stage_bytes = A_BYTES + BN * BK * 2
    for M, clusters in ((1, 1), (129, 1), (1000, 2), (4000, 3)):
        walks = [producer_walk(M, N, K, BN, clusters, r) for r in range(CM)]
        cons = [consumer_walk(M, N, K, BN, clusters, r) for r in range(CM)]
        for c in range(clusters):
            tiles = len(_slots(M, N, BN, clusters, 0)[c])
            seqs = [[e[:3] for e in walks[r][c]] for r in range(CM)]
            # both ranks of the cluster walk the same (stage, phase, kind) sequence, and their consumers wait on exactly it
            assert seqs[0] == seqs[1], (K, BN, M, c)
            assert all(cons[r][c] == seqs[r] for r in range(CM)), (K, BN, M, c)
            assert len(seqs[0]) == tiles * entries
            for i, (_, _, kind) in enumerate(seqs[0]):
                for r in range(CM):
                    own = walks[r][c][i][4]
                    # what lands in rank r's stage: its own loads, and the W boxes the peer loads and multicasts into it
                    peer = {off: v for off, v in walks[1 - r][c][i][4].items() if v[2][0] == "W" and v[1] != r}
                    assert all(own[off] == v for off, v in peer.items()), (K, BN, M, c, i, r)
                    landed = {off: v for off, v in own.items() if v[1] == r} | peer
                    assert sum(nb for nb, _, _ in landed.values()) == walks[r][c][i][3], (K, BN, M, c, i, r)
                    # the boxes of one entry tile its stage without overlap
                    spans = sorted((off, off + nb) for off, (nb, _, _) in landed.items())
                    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] <= stage_bytes
                    if kind == "residual":
                        assert walks[r][c][i][3] == 2 * RES_BOX_BYTES and not peer
        if M == 4000:
            assert len(_slots(M, N, BN, clusters, 0)[0]) > 1  # several tiles per cluster: the ring laps with residual entries in it


# ================================================================================================ GPU: results and launch widths

@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


@gpu
@pytest.mark.parametrize("ln", [False, True], ids=["stats_in NULL", "stats_in"])
@pytest.mark.parametrize("N", [384, 768, 1024])
@pytest.mark.parametrize("K", [64, 192, 768, 3072])
def test_residual_ring_vs_fp64_and_launch_widths(rt, K, N, ln):
    worst = 0.0
    for M in (1, 127, 129, 257, 1000):
        args, kw = _gemm_case(2, M, N, K, seed=K + N + M + ln, ln=ln)
        base = rt.debug_gemm(2, *args, want_stats=True, **kw)
        tag = f"K={K} N={N} M={M} ln={ln}"
        worst = max(worst, KR.check_gemm(tag, base[0], 2, *args, **kw))
        worst = max(worst, KR.check_gemm_stats(tag + " stats_out", base[2], args, **kw))
        for sms in (1, 2, 3):
            got = rt.debug_gemm(2, *args, want_stats=True, sms=sms, **kw)
            assert np.array_equal(got[0].view(np.uint32), base[0].view(np.uint32)), (tag, sms)
            assert np.array_equal(got[2].view(np.uint32), base[2].view(np.uint32)), (tag, sms)
    print(f"K={K} N={N} ln={ln}: worst err/tol {worst:.3f}; sms 1, 2, 3 bitwise equal to every SM")
