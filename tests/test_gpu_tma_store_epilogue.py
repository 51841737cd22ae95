"""The plain fp16 GEMM epilogues (EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_QGELU_F16) stage each consumer warpgroup's 64 rows
of a 64-column chunk in one of two 128B-swizzled [64 x 64] shared-memory boxes and write it with one TMA store through an
{N, M} output map, which clips the rows past M (gemm_sm90.cu, the protocol comment at the top).

Without a GPU: the staging constants are the kernel's; every GEMM instantiation's shared memory fits the 227 KB a CTA may
opt into; and a restatement of the chunk walk covers every (row < M, column) of the output exactly once, issues no box that
lies wholly past M, and never rewrites a staging box whose store may still be reading it -- for M in {1, 63, 64, 65, 127,
128, 129, 8320, 132 * 197} and BN = 256 and 128, over several tiles per cluster.

On the GPU: b200rt.debug_gemm epi 0, 1 and 3 at those M, K in {64, 192, 768, 3072}, BN 256 (N = 512) and 128 (N = 384),
with the LayerNorm folded in where K allows it (768) and without, against the fp64 reference, and bitwise equal at sms = 1,
2, 3 and every SM -- one cluster then walks many tiles with earlier tiles' stores still in flight.  And epi 0 bitwise
equal to the rotary epilogue with no rotated columns, whose register stores do the same arithmetic."""
import os
import re

import numpy as np
import pytest

import instantiations as I
import kernel_refs as KR
from test_gpu_kernels import _gemm_case

gpu = pytest.mark.gpu

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "modal-examples_b200", "csrc", "gemm_sm90.cu")

BM, BK, STAGES, CM = 128, 64, 4, 2
OUT_BOX_BYTES = 64 * 64 * 2
SMEM_LIMIT = 232448  # the dynamic shared memory an sm_90 CTA may opt into
MS = (1, 63, 64, 65, 127, 128, 129, 8320, 132 * 197)
TMA_STORE_EPIS = (I.EPI_BIAS_F16, I.EPI_BIAS_GELU_F16, I.EPI_BIAS_QGELU_F16)


def test_staging_constants_are_the_kernels():
    src = open(SRC).read()
    for name, value in (("BM", BM), ("STAGES", STAGES), ("CM", CM)):
        assert re.search(rf"\b{name} = {value}\b", src), name
    assert re.search(r"\bBK = 64\b", src)
    assert re.search(r"OUT_BOX_BYTES = 64 \* 64 \* 2;", src)
    assert re.search(r"OFF_OUT = OFF_BAR \+ 1024;", src)
    assert re.search(r"OUT_SMEM_BYTES = OFF_OUT \+ 2 \* 2 \* OUT_BOX_BYTES \+ 1024;", src)
    assert re.search(r"tma_store_epi\(int epi\) \{ return epi == EPI_BIAS_F16 \|\| epi == EPI_BIAS_GELU_F16 \|\| epi == EPI_BIAS_QGELU_F16; \}",
                     src)
    assert "tma_store_wait_read<1>();" in src and "tma_store_wait<0>();" in src


def smem_bytes(epi, BN):
    """gemm::smem_bytes<EPI, BN>(): the ring, 1 KB for the barriers (and SPLADE's maxima, or the staging boxes, behind them),
    1 KB of slack to align the dynamic shared memory to 1024."""
    off_bar = STAGES * (BM * BK * 2 + BN * BK * 2)
    if epi == I.EPI_SPLADE_MAX:
        return off_bar + 256 + 1024 + 2 * 4 * BN * 4
    if epi in TMA_STORE_EPIS:
        off_out = off_bar + 1024
        assert off_out % 1024 == 0  # the 128B swizzle's pattern repeats every 1024 bytes
        return off_out + 2 * 2 * OUT_BOX_BYTES + 1024
    return off_bar + 256 + 1024


def test_every_instantiation_fits_shared_memory():
    keys = [k for k in I.REACHABLE if k[0] == I.GEMM]
    assert {k[1] for k in keys} == set(range(7))
    for _, epi, BN, _ in keys:
        assert smem_bytes(epi, BN) <= SMEM_LIMIT, (epi, BN, smem_bytes(epi, BN))
    assert smem_bytes(I.EPI_BIAS_F16, 256) == 231424 and smem_bytes(I.EPI_BIAS_F16, 128) == 165888
    # still one CTA per SM, as before: the staging area does not change the occupancy the kernel was built for
    assert smem_bytes(I.EPI_BIAS_F16, 128) > SMEM_LIMIT // 2


# ================================================================================================ CPU: the chunk walk

def chunk_walk(M, N, BN, clusters):
    """Per cluster, rank and consumer warpgroup: the staging boxes it writes and stores, in order, as (box, column, row, rows
    written after the map clips them).  A warpgroup whose 64 rows all lie past M writes and stores nothing."""
    num_n = N // BN
    num_slots = -(-M // (CM * BM)) * num_n * CM
    walks = {}
    for c in range(clusters):
        for rank in range(CM):
            for cw in range(2):
                seq = []
                for t in range(CM * c + rank, num_slots, CM * clusters):
                    p = t // CM
                    m0, n0 = ((p // num_n) * CM + t % CM) * BM, (p % num_n) * BN
                    row = m0 + 64 * cw
                    if row < M:
                        seq += [(q % 2, n0 + 64 * q, row, min(64, M - row)) for q in range(BN // 64)]
                walks[c, rank, cw] = seq
    return walks


@pytest.mark.parametrize("BN", [256, 128])
@pytest.mark.parametrize("M", MS)
def test_chunk_walk_covers_every_row_below_m_once(M, BN):
    N = 3 * BN
    for clusters in (1, 3, 66):
        hits = np.zeros((M, N), np.int32)
        for seq in chunk_walk(M, N, BN, clusters).values():
            pending = []  # the issuer's bulk groups not yet known to have read their box
            for box, col, row, rows in seq:
                pending = pending[-1:]  # cp.async.bulk.wait_group.read 1
                assert box not in pending, (M, BN, clusters)
                assert 0 < rows <= 64 and row < M  # no box issued wholly past M
                hits[row:row + rows, col:col + 64] += 1
                pending.append(box)
        assert (hits == 1).all(), (M, BN, clusters)


# ================================================================================================ GPU

@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.init(devices=[0])
    yield b200rt
    b200rt.shutdown()


@gpu
# the folded LayerNorm is 768, 384 or 1024 wide: of these K, 768 only takes it
@pytest.mark.parametrize("K,ln", [(64, False), (192, False), (768, False), (768, True), (3072, False)])
@pytest.mark.parametrize("N", [512, 384], ids=["BN 256", "BN 128"])
@pytest.mark.parametrize("epi", TMA_STORE_EPIS)
def test_tma_store_epilogue_vs_fp64_and_launch_widths(rt, epi, N, K, ln):
    worst = 0.0
    for M in MS:
        args, kw = _gemm_case(epi, M, N, K, seed=7 * epi + K + N + M + ln, ln=ln)
        base = rt.debug_gemm(epi, *args, **kw)[0]
        tag = f"epi {epi} N={N} K={K} M={M} ln={ln}"
        worst = max(worst, KR.check_gemm(tag, base.astype(np.float64), epi, *args, **kw))
        for sms in (1, 2, 3):
            got = rt.debug_gemm(epi, *args, sms=sms, **kw)[0]
            assert np.array_equal(got.view(np.uint16), base.view(np.uint16)), (tag, sms)
    print(f"epi {epi} N={N} K={K} ln={ln}: worst err/tol {worst:.3f}; sms 1, 2, 3 bitwise equal to every SM")


@gpu
@pytest.mark.parametrize("ln", [False, True], ids=["stats_in NULL", "stats_in"])
@pytest.mark.parametrize("M", [64, 8320])
def test_tma_store_matches_register_store_epilogue(rt, M, ln):
    """EPI_ROPE_F16 with rot_cols = 0 rotates nothing: each tile takes its V branch, rstd * acc + c stored from registers
    with the same arithmetic as EPI_BIAS_F16, so the two outputs are bitwise equal."""
    N, K, S = 2304, 768, 64
    args, kw = _gemm_case(0, M, N, K, seed=M + ln, ln=ln)
    a, w, bias = args
    st = kw.get("ln_stats")
    got = rt.debug_gemm(0, *args, **kw)[0]
    table = np.zeros((S, 32, 2), np.float32)
    want = rt.debug_gemm_rope(a, w, bias, st, table, S, 0, kw["eps"])
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
