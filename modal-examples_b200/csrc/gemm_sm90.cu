// Warp-specialised wgmma GEMM for sm_90a:  C[M,N] = epilogue(A[M,K] . W[N,K]^T + bias)
//
// Persistent clusters of CM = 2 CTAs walk pairs of 128 x BN output tiles that share their columns, BN = 256, or 128 where
// N % 256 != 0 (bge-small's 384 / 1152-wide projections; the figures below are BN = 256's, BN = 128 halves the W box, the
// stage and the accumulators).  The LayerNorm statistics a tile reads come as PARTS partials per row: 6 (768 wide), 3 (384),
// 8 (bge-large's 1024) or 4 (the CLIP text tower's 512).  Pair p = (m-pair p / num_n, n-block p % num_n), n fastest; CTA rank r of the cluster takes
// m-tile CM (p / num_n) + r; cluster c walks p = c, c + clusters, ..., its two CTAs in step.  Three warpgroups per CTA:
//   warpgroup 0  : one thread TMA-loads its own A [128 x 64] per 64-wide k-block into a STAGES-deep ring (48 KB per stage,
//                  128B-swizzled), plus its share of the pair's W [256 x 64] -- 128-row box b is loaded by rank b % CM and
//                  multicast into the same stage of every CTA of the cluster, so the pair reads W from L2 once instead of
//                  twice (2 A + W = 64 KB per k-block-pair instead of 96 KB).  It runs ahead across tiles while the
//                  consumers are in their epilogue;
//   warpgroups 1-2: consumer c owns rows 64c .. 64c+63 of the tile and all 256 columns: four wgmma.m64n256k16 per k-block
//                  into 128 fp32 accumulator registers per thread, one k-block's MMAs kept in flight while the previous
//                  stage is handed back to the producers; then the epilogue runs from the registers (EPI_BIAS(_GELU /
//                  _QGELU)_F16: into shared memory, and TMA stores it, see below).
//
//   full[s]  : own producer arrive.expect_tx(48 KB); own A, own W share and the peer's W share complete_tx on it
//   empty[s] : one arrival per consumer warp of EVERY CTA of the cluster once the wgmma that read stage s have completed
//              (8 CM arrivals): a producer refills a stage -- its multicast writes the peer's copy too -- only once the
//              consumers of both CTAs are done with it.  Both CTAs walk the same pairs and k-blocks, so the rings run in
//              lockstep.  A rank whose m-tile lies past M still loads and arrives; its epilogue stores nothing (row < M).
// A cluster barrier after the barrier init (before any remote arrive or multicast) and one before exit (so that no CTA leaves
// while the peer may still arrive on its barriers) bracket the protocol; every thread of both warpgroups takes both.
//
// EPI_BIAS_RES_SPLIT brings the tile's residual in through the same ring: after the tile's last k-block the producer takes
// BN / 64 more entries, one per 64-column chunk q, each the hi box [128 rows x 64 columns] at (n0 + 64q, m0) at the stage's
// offset 0 and the lo box at 16 KB (expect_tx 32 KB; own rows only, not multicast).  The consumers wait on full[s], read the
// chunk from shared memory, store it and arrive on empty[s] exactly as for an operand stage (8 CM arrivals).  Both CTAs walk
// the same pairs with the same K and BN, so both add the same entries at the same points and the rings stay in lockstep; a
// tile past M loads the map's rows there or out-of-bounds zeros, with the full byte count either way, and stores nothing.
// Each thread writes hi' and lo' over the very values it read; a named barrier over the consumer warpgroup then lets its 128
// threads copy the warpgroup's 64 rows of the chunk to global memory as 16-byte pieces of whole 128-byte rows (rows < M).
//   * The stage is read and written by the generic proxy (ld/st.shared), and its next write is a TMA (async proxy) of this
//     CTA's producer or, for a W box, the peer's.  Every consumer thread issues fence.proxy.async after its last access,
//     so its shared-memory writes are ordered before any later async-proxy write; its reads have returned their values
//     (they were stored to global memory) before the __syncwarp ahead of its warp's arrive; the arrive releases both, and a
//     producer issues the TMA only after its wait on empty[s] has acquired all 8 CM arrivals.
//   * Each element of y is written in place by the one tile that owns it, after that tile's TMA has read it (the consumer
//     stores only after its wait on full[s] saw the read complete).  Tiles are disjoint, so no tile reads what another wrote.
//
// EPI_BIAS(_GELU / _QGELU)_F16 store their output by TMA through a staging area behind the barriers, outside the ring: two
// [64 rows x 64 columns] fp16 boxes (8 KB, 128B-swizzled) per consumer warpgroup.  For each 64-column chunk q of the tile the
// warpgroup writes its 64 rows of the chunk into box q % 2, and its first thread (the issuer) stores the box to (n0 + 64q,
// m0 + 64 cw) with one TMA store and commits it as one bulk group.  Nothing waits for the stores to land: the warpgroup goes
// on to its next chunk and its next tile's main loop while the TMA engine drains them.  A warpgroup whose 64 rows all lie
// past M writes no box and stores nothing.
//   * The output map is {N, M}: exactly M rows, so TMA clips a box's rows past M and rows past M are never written.
//   * Before box q % 2 is rewritten, the issuer's cp.async.bulk.wait_group.read 1 leaves only the other box's store (chunk
//     q - 1) pending, so the store of chunk q - 2 has finished reading it; a named barrier over the warpgroup then lets its
//     128 threads write.  BN / 64 is even and a tile stores all of its chunks or none, so every store's box alternates
//     with the one before it across tiles as well.
//   * Every thread issues fence.proxy.async after its writes (generic proxy) and before a second named barrier, after
//     which the issuer's TMA (async proxy) reads the box.
//   * The issuer waits for all its stores to complete (cp.async.bulk.wait_group 0) before the final cluster barrier: the
//     staging area must outlive their reads, and the output must be in global memory when the grid ends, since the next
//     kernel's griddepcontrol.wait only waits for the grid.
//
// Epilogues (see kernels.h for the residual-stream format):
//   EPI_BIAS(_GELU / _QGELU)_F16 : folded LayerNorm  rstd * acc + c  (c = W beta + b), optional GELU, fp16 out;
//   EPI_BIAS_RES_SPLIT           : y' = acc + bias + LN(y) with the LayerNorm re-applied from the row's statistics, y' split
//                                  into fp16 hi + lo in place, and the (sum, M2) partial of each new 128-column row slice;
//   EPI_SPLADE_MAX               : v = max(rstd * acc + c, 0) on the item's valid rows, max-reduced over the consumer's 64 rows
//                                  (one item: S % 64 == 0) by shuffles and a 4 KB shared-memory pass, then one
//                                  red.global.max.u32 per non-zero column < vocab into the item's row of the max buffer;
//   EPI_ROPE_F16                 : v = rstd * acc + c as EPI_BIAS_F16, then on columns < rp.rot_cols (Q and K) each pair
//                                  (d, d + 32) of a 64-column head rotated by the angle of position row % rp.S; fp16 out;
//   EPI_SWIGLU_F16               : W's rows are gate and up interleaved in 8-row groups (g on 16k .. 16k+7, u on 16k+8 ..
//                                  16k+15), so accumulator groups 2m and 2m+1 hold matching g and u columns: fp16(silu(g) u)
//                                  into out [M, N / 2].
//
// The accumulator fragment of thread (warp w of the consumer warpgroup, lane l) holds rows 16w + l/4 and 16w + l/4 + 8,
// columns 8j + 2(l%4) + {0, 1} for j = 0..31: acc[4j + {0, 1}] on the first row, acc[4j + {2, 3}] on the second.
//
// Replaces (inside TEI, un-vendored; restated from HF modeling_bert.py): the Linear layers of
// BertSelfAttention :143-207 (fused QKV), BertSelfOutput.dense :287-298, BertIntermediate :330-342
// (dense + GELU) and BertOutput.dense :345-356.
#include <algorithm>
#include <tuple>

#include "kernels.h"
#include "ptx.cuh"

namespace b200 {
namespace gemm {

constexpr int BM = 128;  // rows per tile (two consumer warpgroups of 64)
constexpr int BK = 64, STAGES = 4;
constexpr int A_BYTES = BM * BK * 2;            // 16 KB
constexpr int W_BOX_BYTES = 128 * BK * 2;       // one 128-row TMA box of W: 16 KB
constexpr int NUM_THREADS = 384;
constexpr int CM = 2;  // CTAs per cluster, along M, sharing every W tile
constexpr int RES_BOX_BYTES = BM * 64 * 2;      // EPI_BIAS_RES_SPLIT: one [128 x 64] box of hi or lo, 16 KB
constexpr int OUT_BOX_BYTES = 64 * 64 * 2;      // EPI_BIAS(_GELU / _QGELU)_F16: one [64 x 64] staging box of the output, 8 KB

// the epilogues that stage their fp16 output in shared memory and store it by TMA
constexpr bool tma_store_epi(int epi) { return epi == EPI_BIAS_F16 || epi == EPI_BIAS_GELU_F16 || epi == EPI_BIAS_QGELU_F16; }

// ring layout of the BN-column kernel
template <int BN>
struct Tiles {
    static constexpr int B_BYTES = BN * BK * 2;            // 32 KB (two TMA boxes of 128 rows) / 16 KB (one)
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;  // 48 KB / 32 KB
    static constexpr int OFF_BAR = STAGES * STAGE_BYTES;
    static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
    static_assert(SMEM_BYTES <= 232448, "shared memory");
    // EPI_SPLADE_MAX: behind the barriers, each consumer warpgroup's [4 warps][BN] column maxima
    static constexpr int OFF_RED = OFF_BAR + 256;
    static constexpr int SPLADE_SMEM_BYTES = SMEM_BYTES + 2 * 4 * BN * 4;
    static_assert(SPLADE_SMEM_BYTES <= 232448, "shared memory");
    // tma_store_epi: behind the barriers, 1024-aligned for the 128B swizzle, each consumer warpgroup's two staging boxes
    static constexpr int OFF_OUT = OFF_BAR + 1024;
    static constexpr int OUT_SMEM_BYTES = OFF_OUT + 2 * 2 * OUT_BOX_BYTES + 1024;  // 231 424 / 165 888
    static_assert(OUT_SMEM_BYTES <= 232448, "shared memory");
};
template <int EPI, int BN>
constexpr int smem_bytes() {
    return EPI == EPI_SPLADE_MAX ? Tiles<BN>::SPLADE_SMEM_BYTES : tma_store_epi(EPI) ? Tiles<BN>::OUT_SMEM_BYTES : Tiles<BN>::SMEM_BYTES;
}

// erf-GELU x * Phi(x), erf by Abramowitz-Stegun 7.1.26 (abs err <= 1.5e-7): 2 MUFU (rcp, ex2) per value
__device__ __forceinline__ float gelu_erf(float x) {
    const float a = fabsf(x);
    const float u = fmaf(a, 0.3275911f * 0.70710678118654752f, 1.0f);
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(u));
    float p = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
    p = fmaf(p, t, 0.5f * 1.421413741f);
    p = fmaf(p, t, 0.5f * -0.284496736f);
    p = fmaf(p, t, 0.5f * 0.254829592f);
    const float q = p * t * ex2_approx(a * (-0.5f * 1.4426950408889634f) * a);
    return x * (x >= 0.f ? 1.0f - q : q);
}

// CLIP's quick_gelu: x * sigmoid(1.702 x) = x / (1 + 2^(-1.702 log2(e) x))
__device__ __forceinline__ float gelu_quick(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(ex2_approx(x * (-1.702f * 1.4426950408889634f)) + 1.0f));
    return x * r;
}

// silu(g) = g / (1 + 2^(-g log2(e))): ex2.approx (relative error <= 2^-22) and rcp.approx (<= 1 ulp) put the result within
// 4e-7 relative of silu(g) wherever it is finite and non-zero -- three orders of magnitude inside fp16's half ulp (2^-12).  For
// g < -88 the exponential overflows to +inf, rcp gives 0 and silu(g) = -0 (the true value is below 1e-36).
__device__ __forceinline__ float silu(float g) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(ex2_approx(g * -1.4426950408889634f) + 1.0f));
    return g * r;
}

// LayerNorm statistics of a row from its PARTS (sum, M2) partials (Chan et al.): 8 for a 1024-wide row, 6 for a 768-wide one,
// 4 for a 512-wide one, 3 for a 384-wide one
template <int PARTS>
__device__ __forceinline__ void row_stats(const float2* __restrict__ st, float eps, float& mean, float& rstd) {
    static_assert(PARTS == 8 || PARTS == 6 || PARTS == 4 || PARTS == 3, "LayerNorm width 1024, 768, 512 or 384");
    constexpr float inv_n = 1.0f / (128.0f * PARTS);
    if constexpr (PARTS == 8) {
        const float4* __restrict__ pp = reinterpret_cast<const float4*>(st);
        const float4 a = __ldg(pp), b = __ldg(pp + 1), c = __ldg(pp + 2), d = __ldg(pp + 3);
        const float2 p[PARTS] = {make_float2(a.x, a.y), make_float2(a.z, a.w), make_float2(b.x, b.y), make_float2(b.z, b.w),
                                 make_float2(c.x, c.y), make_float2(c.z, c.w), make_float2(d.x, d.y), make_float2(d.z, d.w)};
        mean = (((p[0].x + p[1].x) + (p[2].x + p[3].x)) + ((p[4].x + p[5].x) + (p[6].x + p[7].x))) * inv_n;
        float m2[PARTS];
#pragma unroll
        for (int i = 0; i < PARTS; ++i) {
            const float d = p[i].x * (1.0f / 128.0f) - mean;
            m2[i] = fmaf(128.0f * d, d, p[i].y);
        }
        rstd = rsqrtf((((m2[0] + m2[1]) + (m2[2] + m2[3])) + ((m2[4] + m2[5]) + (m2[6] + m2[7]))) * inv_n + eps);
    } else if constexpr (PARTS == 6) {
        const float4* __restrict__ pp = reinterpret_cast<const float4*>(st);
        const float4 a = __ldg(pp), b = __ldg(pp + 1), c = __ldg(pp + 2);
        const float2 p[PARTS] = {make_float2(a.x, a.y), make_float2(a.z, a.w), make_float2(b.x, b.y),
                                 make_float2(b.z, b.w), make_float2(c.x, c.y), make_float2(c.z, c.w)};
        mean = (((p[0].x + p[1].x) + (p[2].x + p[3].x)) + (p[4].x + p[5].x)) * inv_n;
        float m2[PARTS];
#pragma unroll
        for (int i = 0; i < PARTS; ++i) {
            const float d = p[i].x * (1.0f / 128.0f) - mean;
            m2[i] = fmaf(128.0f * d, d, p[i].y);
        }
        rstd = rsqrtf((((m2[0] + m2[1]) + (m2[2] + m2[3])) + (m2[4] + m2[5])) * inv_n + eps);
    } else if constexpr (PARTS == 4) {
        // a pairwise tree, as for 8
        const float4* __restrict__ pp = reinterpret_cast<const float4*>(st);
        const float4 a = __ldg(pp), b = __ldg(pp + 1);
        const float2 p[PARTS] = {make_float2(a.x, a.y), make_float2(a.z, a.w), make_float2(b.x, b.y), make_float2(b.z, b.w)};
        mean = ((p[0].x + p[1].x) + (p[2].x + p[3].x)) * inv_n;
        float m2[PARTS];
#pragma unroll
        for (int i = 0; i < PARTS; ++i) {
            const float d = p[i].x * (1.0f / 128.0f) - mean;
            m2[i] = fmaf(128.0f * d, d, p[i].y);
        }
        rstd = rsqrtf(((m2[0] + m2[1]) + (m2[2] + m2[3])) * inv_n + eps);
    } else {
        // a row's three partials are 24 bytes: 8-byte loads
        const float2 p[PARTS] = {__ldg(st), __ldg(st + 1), __ldg(st + 2)};
        mean = ((p[0].x + p[1].x) + p[2].x) * inv_n;
        float m2[PARTS];
#pragma unroll
        for (int i = 0; i < PARTS; ++i) {
            const float d = p[i].x * (1.0f / 128.0f) - mean;
            m2[i] = fmaf(128.0f * d, d, p[i].y);
        }
        rstd = rsqrtf(((m2[0] + m2[1]) + m2[2]) * inv_n + eps);
    }
}

// BN: tile width (256 or 128); PARTS: partials per row of ep.stats_in (the LayerNorm'd width / 128).  sp is read by
// EPI_SPLADE_MAX only, rp by EPI_ROPE_F16 only, res by EPI_BIAS_RES_SPLIT only, oe by tma_store_epi only; as the last
// parameters they leave every other instantiation's parameter offsets as they were.
template <int EPI, int BN, int PARTS>
__global__ void __cluster_dims__(CM, 1, 1) __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const GemmEpi ep,
            __half* __restrict__ out, __half* __restrict__ out_lo, int M, int N, int K, const SpladeEpi sp, const RopeEpi rp,
            const __grid_constant__ ResEpi res, const __grid_constant__ OutEpi oe) {
    static_assert(BN == 256 || BN == 128, "tile width");
    constexpr int STAGE_BYTES = Tiles<BN>::STAGE_BYTES, OFF_BAR = Tiles<BN>::OFF_BAR;
    constexpr int NACC = BN / 2;     // fp32 accumulators per consumer thread
    constexpr int NSLICE = BN / 128; // 128-column statistic slices per tile, and 128-row W boxes per stage
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* full = bars;            // [STAGES]
    uint64_t* empty = bars + STAGES;  // [STAGES]

    griddep_launch_dependents();
    const int warp = __shfl_sync(0xffffffff, threadIdx.x >> 5, 0);
    const int lane = lane_id();
    const int num_n = N / BN;
    // Slot t = CM p + r is rank r's tile of pair p.  A 1-D grid of (CM, 1, 1) clusters numbers its CTAs blockIdx.x =
    // CM cluster + rank, so t = blockIdx.x, blockIdx.x + gridDim.x, ... walks pairs cluster, cluster + clusters, ... with both
    // ranks in step (and keeps the loop state of an unclustered walk: two more live registers spill the epilogue).
    const int num_slots = ((M + CM * BM - 1) / (CM * BM)) * num_n * CM;
    const int kblocks = K / BK;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tma_a);
        prefetch_tmap(&tma_b);
        if constexpr (EPI == EPI_BIAS_RES_SPLIT) {
            prefetch_tmap(&res.hi);
            prefetch_tmap(&res.lo);
        }
        if constexpr (tma_store_epi(EPI)) prefetch_tmap(&oe.out);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8 * CM);  // the 8 consumer warps of every CTA of the cluster
        }
        fence_barrier_init();
    }
    cluster_sync();  // the peer's barriers are initialised before anything arrives on them or multicasts into its ring
    griddep_wait();  // everything above overlapped the previous kernel's tail; nothing it wrote has been read yet

    if (warp < 4) {
        // -------------------------------------------------------------------- TMA producer
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_slots; t += gridDim.x) {
                const int p = t / CM, rank = t % CM;
                const int m0 = ((p / num_n) * CM + rank) * BM, n0 = (p % num_n) * BN;
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);  // the consumers of every CTA of the cluster have freed the stage
                    uint8_t* sa = smem + stage * STAGE_BYTES;
                    mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);  // own A + all of W, whichever CTA loads each box
                    tma_load_2d(sa, &tma_a, &full[stage], kb * BK, m0);
                    for (int b = rank; b < NSLICE; b += CM)
                        tma_load_2d_multicast(sa + A_BYTES + b * W_BOX_BYTES, &tma_b, &full[stage], kb * BK, n0 + 128 * b,
                                              (1u << CM) - 1);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
                if constexpr (EPI == EPI_BIAS_RES_SPLIT) {
                    for (int q = 0; q < BN / 64; ++q) {  // the tile's residual, one 64-column chunk of hi and lo per entry
                        mbar_wait(&empty[stage], phase ^ 1);
                        uint8_t* sr = smem + stage * STAGE_BYTES;
                        mbar_arrive_expect_tx(&full[stage], 2 * RES_BOX_BYTES);
                        tma_load_2d(sr, &res.hi, &full[stage], n0 + 64 * q, m0);
                        tma_load_2d(sr + RES_BOX_BYTES, &res.lo, &full[stage], n0 + 64 * q, m0);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        __syncwarp();
        cluster_sync();
        return;
    }

    // ------------------------------------------------------------------------ consumers
    setmaxnreg_inc<232>();
    const int cw = (warp >> 2) - 1;  // which 64 rows of the tile
    const int w4 = warp & 3;
    const float* __restrict__ bias = ep.bias;
    const bool has_ln = ep.stats_in != nullptr;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < num_slots; t += gridDim.x) {
        const int p = t / CM;
        const int m0 = ((p / num_n) * CM + t % CM) * BM, n_blk = p % num_n, n0 = n_blk * BN;
        float acc[NACC];
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint32_t a_addr = smem_u32(smem + stage * STAGE_BYTES) + cw * (64 * 128);
            const uint32_t b_addr = smem_u32(smem + stage * STAGE_BYTES) + A_BYTES;
            wgmma_fence();
            fence_operands(acc);
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                if constexpr (BN == 256) wgmma_m64n256k16_ss(acc, make_sw128_desc(a_addr + k * 32), make_sw128_desc(b_addr + k * 32), (kb | k) != 0);
                else wgmma_m64n128k16_ss(acc, make_sw128_desc(a_addr + k * 32), make_sw128_desc(b_addr + k * 32), (kb | k) != 0);
            }
            wgmma_commit();
            fence_operands(acc);
            if (prev >= 0) {
                wgmma_wait<1>();  // the previous k-block's MMAs have read their stage
                if (lane < CM) mbar_arrive_cluster(&empty[prev], lane);  // lane r frees it in CTA r's producer's eyes
            }
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_operands(acc);
        if (lane < CM) mbar_arrive_cluster(&empty[prev], lane);

        // -------------------------------------------------------------------- epilogue, straight from the registers
        const int r0 = m0 + cw * 64 + w4 * 16 + (lane >> 2);  // this thread's rows r0 and r0 + 8
        const int c0 = n0 + 2 * (lane & 3);                   // its columns c0 + 8j + {0, 1}
        float mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
        if (has_ln) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (r0 + 8 * h < M) row_stats<PARTS>(ep.stats_in + static_cast<size_t>(r0 + 8 * h) * PARTS, ep.eps, mean[h], rstd[h]);
        }
        if constexpr (EPI == EPI_SPLADE_MAX) {
            // the consumer's 64 rows hrow0 .. hrow0 + 63 lie in item hrow0 / S (S % 64 == 0, M = B S); `valid` of them, from
            // hrow0 on, are inside the item's length -- the same for every thread of the warpgroup
            const int hrow0 = m0 + cw * 64;
            const int item = hrow0 / sp.S;
            const int valid = hrow0 < M ? min(max(__ldg(sp.lens + item), 0), sp.S) - (hrow0 - item * sp.S) : 0;
            if (valid > 0) {
                float* red = reinterpret_cast<float*>(smem + Tiles<BN>::OFF_RED) + cw * (4 * BN);  // [warp][column]
                const int lr = w4 * 16 + (lane >> 2);  // this thread's rows within the half: lr and lr + 8
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + c0 + 8 * j));
                    float v0 = 0.f, v1 = 0.f;  // relu: the max starts at 0
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (lr + 8 * h < valid) {
                            v0 = fmaxf(v0, fmaf(rstd[h], acc[4 * j + 2 * h], bv.x));
                            v1 = fmaxf(v1, fmaf(rstd[h], acc[4 * j + 2 * h + 1], bv.y));
                        }
                    // the 8 lanes of a warp that hold these two columns differ in lane bits 2..4
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        v0 = fmaxf(v0, __shfl_xor_sync(0xffffffff, v0, o));
                        v1 = fmaxf(v1, __shfl_xor_sync(0xffffffff, v1, o));
                    }
                    if (lane < 4) *reinterpret_cast<float2*>(red + w4 * BN + 8 * j + 2 * lane) = make_float2(v0, v1);
                }
                named_bar_sync(1 + cw, 128);
                const int t = threadIdx.x - 128 * (cw + 1);
                uint32_t* vrow = sp.vmax + static_cast<size_t>(item) * N;
#pragma unroll
                for (int cl = t; cl < BN; cl += 128) {
                    const float v = fmaxf(fmaxf(red[cl], red[BN + cl]), fmaxf(red[2 * BN + cl], red[3 * BN + cl]));
                    // values are >= 0, so the integer max of the fp32 bits is the float max, in any order
                    if (v > 0.f && n0 + cl < sp.vocab) atomicMax(vrow + n0 + cl, __float_as_uint(v));
                }
                named_bar_sync(1 + cw, 128);  // the next tile rewrites red
            }
        } else if constexpr (EPI == EPI_ROPE_F16) {
            // head column d < 32 of accumulator group j = 8 hh + jj (jj < 4) pairs with d + 32 in group j + 4 of the same thread;
            // both take frequency d = 8 jj + 2 (lane % 4) + {0, 1}: one float4 (cos, sin, cos, sin) per row and jj.  Q / K / V
            // boundaries fall on tile boundaries, so a tile is rotated whole (Q, K) or not at all (V).  S % 64 == 0, so the
            // consumer's 64 rows are positions (m0 + 64 cw) % S on and this thread's two rows lie 8 positions apart.
            if (n0 < rp.rot_cols) {
                const float4* __restrict__ cs = reinterpret_cast<const float4*>(rp.table) +
                                                ((m0 + cw * 64) % rp.S + w4 * 16 + (lane >> 2)) * 16 + (lane & 3);
#pragma unroll
                for (int hh = 0; hh < BN / 64; ++hh) {  // head by head; the table row is re-read (L1) for each
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int j0 = 8 * hh + jj, j1 = j0 + 4;
                        const float2 b0 = __ldg(reinterpret_cast<const float2*>(bias + c0 + 8 * j0));
                        const float2 b1 = __ldg(reinterpret_cast<const float2*>(bias + c0 + 8 * j1));
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int row = r0 + 8 * h;
                            if (row >= M) continue;
                            const float4 t = __ldg(cs + 128 * h + 4 * jj);
                            const float x0 = fmaf(rstd[h], acc[4 * j0 + 2 * h], b0.x), x1 = fmaf(rstd[h], acc[4 * j0 + 2 * h + 1], b0.y);
                            const float y0 = fmaf(rstd[h], acc[4 * j1 + 2 * h], b1.x), y1 = fmaf(rstd[h], acc[4 * j1 + 2 * h + 1], b1.y);
                            // x_d cos - x_{d+32} sin,  x_{d+32} cos + x_d sin
                            __half* o = out + static_cast<size_t>(row) * N + c0;
                            *reinterpret_cast<uint32_t*>(o + 8 * j0) = pack_half2(fmaf(x0, t.x, -y0 * t.y), fmaf(x1, t.z, -y1 * t.w));
                            *reinterpret_cast<uint32_t*>(o + 8 * j1) = pack_half2(fmaf(y0, t.x, x0 * t.y), fmaf(y1, t.z, x1 * t.w));
                        }
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + c0 + 8 * j));
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = r0 + 8 * h;
                        if (row < M)
                            *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(row) * N + c0 + 8 * j) =
                                pack_half2(fmaf(rstd[h], acc[4 * j + 2 * h], bv.x), fmaf(rstd[h], acc[4 * j + 2 * h + 1], bv.y));
                    }
                }
            }
        } else if constexpr (EPI == EPI_SWIGLU_F16) {
            // groups 2m (gate) and 2m + 1 (up) -> output columns n0 / 2 + 8m + 2 (lane % 4) + {0, 1} of the N / 2 wide rows
#pragma unroll
            for (int m = 0; m < BN / 16; ++m) {
                const float2 bg = __ldg(reinterpret_cast<const float2*>(bias + c0 + 16 * m));
                const float2 bu = __ldg(reinterpret_cast<const float2*>(bias + c0 + 16 * m + 8));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float g0 = fmaf(rstd[h], acc[8 * m + 2 * h], bg.x), g1 = fmaf(rstd[h], acc[8 * m + 2 * h + 1], bg.y);
                    const float u0 = fmaf(rstd[h], acc[8 * m + 4 + 2 * h], bu.x), u1 = fmaf(rstd[h], acc[8 * m + 4 + 2 * h + 1], bu.y);
                    const int row = r0 + 8 * h;
                    if (row < M)
                        *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(row) * (N / 2) + n0 / 2 + 8 * m + 2 * (lane & 3)) =
                            pack_half2(silu(g0) * u0, silu(g1) * u1);
                }
            }
        } else if constexpr (EPI != EPI_BIAS_RES_SPLIT) {
            // one 64-column chunk q at a time through staging box q % 2 (see the top of the file): this thread's rows of the box
            // are lr and lr + 8, and 128B swizzle puts 16-byte column group jj of box row r at (jj ^ r % 8) * 16 -- r % 8 =
            // lane / 4 for both rows, so a warp's 32 writes fall in 32 distinct banks
            const bool issuer = (threadIdx.x & 127) == 0;
            const int lr = w4 * 16 + (lane >> 2);
            uint8_t* const stg = smem + Tiles<BN>::OFF_OUT + cw * (2 * OUT_BOX_BYTES);
            if (m0 + 64 * cw < M) {
#pragma unroll
                for (int q = 0; q < BN / 64; ++q) {
                    uint8_t* const box = stg + (q & 1) * OUT_BOX_BYTES;
                    if (issuer) tma_store_wait_read<1>();  // the store of chunk q - 2 has read the box
                    named_bar_sync(1 + cw, 128);
                    const uint32_t row_addr = smem_u32(box) + lr * 128 + 4 * (lane & 3);
#pragma unroll
                    for (int j = 8 * q; j < 8 * q + 8; ++j) {
                        const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + c0 + 8 * j));
                        const uint32_t a = row_addr + (static_cast<uint32_t>((j & 7) ^ (lane >> 2)) << 4);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            // folded LayerNorm: rstd * acc + c -- the weight rows are centred at load time (sum_k W''[n,k] = 0),
                            // so the row mean cancels inside the tensor core: sum_k (y_k - mean) W''_nk = sum_k y_k W''_nk
                            float v0 = fmaf(rstd[h], acc[4 * j + 2 * h], bv.x);
                            float v1 = fmaf(rstd[h], acc[4 * j + 2 * h + 1], bv.y);
                            if constexpr (EPI == EPI_BIAS_GELU_F16) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
                            if constexpr (EPI == EPI_BIAS_QGELU_F16) { v0 = gelu_quick(v0); v1 = gelu_quick(v1); }
                            sts32(a + h * (8 * 128), pack_half2(v0, v1));
                        }
                    }
                    fence_proxy_async_smem();     // the writes are ordered before the TMA store's reads
                    named_bar_sync(1 + cw, 128);  // the warpgroup's 64 rows of the chunk are in the box
                    if (issuer) {
                        tma_store_2d(&oe.out, box, n0 + 64 * q, m0 + 64 * cw);
                        tma_store_commit();
                    }
                }
            }
        } else {
            // y' = acc + bias + LN(y); LN(y) = fmaf((y - mean) * rstd, gamma, beta) (stats_in NULL: the residual is added as is)
            float csum[2][NSLICE] = {};  // [row][128-column slice of the tile]
#pragma unroll
            for (int q = 0; q < BN / 64; ++q) {
                // the ring entry of columns n0 + 64q ..: this thread's rows of the boxes are 64 cw + 16 w4 + lane / 4 + 8 h, and
                // 128B swizzle puts 16-byte column group jj of box row r at (jj ^ r % 8) * 16 -- r % 8 = lane / 4 for both rows,
                // so a warp's 32 reads fall in 32 distinct banks.  hi' and lo' go back over the values they replace, and the
                // warpgroup then stores its 64 rows of the chunk as whole 128-byte rows instead of 4-byte fragments.
                mbar_wait(&full[stage], phase);
                const uint32_t sbase = smem_u32(smem + stage * STAGE_BYTES);
                const uint32_t box = sbase + (cw * 64 + w4 * 16 + (lane >> 2)) * 128 + 4 * (lane & 3);
#pragma unroll
                for (int j = 8 * q; j < 8 * q + 8; ++j) {
                    const int col = c0 + 8 * j;
                    const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + col));
                    float2 gm = make_float2(1.f, 1.f), bt = make_float2(0.f, 0.f);
                    if (has_ln) {
                        gm = __ldg(reinterpret_cast<const float2*>(ep.ln_gamma + col));
                        bt = __ldg(reinterpret_cast<const float2*>(ep.ln_beta + col));
                    }
                    const uint32_t sw = static_cast<uint32_t>((j & 7) ^ (lane >> 2)) << 4;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = r0 + 8 * h;
                        float& v0 = acc[4 * j + 2 * h];
                        float& v1 = acc[4 * j + 2 * h + 1];
                        if (row < M) {
                            const uint32_t a = box + h * (8 * 128) + sw;
                            const float2 hv = __half22float2(lds_half2(a));
                            const float2 lv = __half22float2(lds_half2(a + RES_BOX_BYTES));
                            v0 = v0 + bv.x + fmaf((hv.x + lv.x - mean[h]) * rstd[h], gm.x, bt.x);
                            v1 = v1 + bv.y + fmaf((hv.y + lv.y - mean[h]) * rstd[h], gm.y, bt.y);
                            // split y' = hi' + lo'
                            const __half2 hp = __floats2half2_rn(v0, v1);
                            const float2 hb = __half22float2(hp);
                            sts32(a, *reinterpret_cast<const uint32_t*>(&hp));
                            sts32(a + RES_BOX_BYTES, pack_half2(v0 - hb.x, v1 - hb.y));
                        }
                        csum[h][j >> 4] += v0 + v1;
                    }
                }
                named_bar_sync(1 + cw, 128);  // the warpgroup's 64 rows of hi' and lo' are in the stage
                {
                    // 128 threads x 16 bytes: 16 rows per pass, a warp covering 4 whole rows; unit u = row 8 + column group
                    const int t = threadIdx.x - 128 * (cw + 1);
#pragma unroll 1
                    for (int pass = 0; pass < 8; ++pass) {  // rolled: the 128 accumulators leave room for one value in flight
                        const int u = (pass & 3) * 128 + t, lr = u >> 3, cg = u & 7;
                        const int row = m0 + cw * 64 + lr;
                        const uint32_t a = sbase + (pass >> 2) * RES_BOX_BYTES + (cw * 64 + lr) * 128 + ((cg ^ (lr & 7)) << 4);
                        const uint4 v = lds128(a);
                        if (row < M)
                            *reinterpret_cast<uint4*>(((pass >> 2) ? out_lo : out) + static_cast<size_t>(row) * N + n0 + 64 * q + 8 * cg) = v;
                    }
                }
                // every lane's reads of the stage are done, and its shared-memory writes ordered before the TMA that will
                // overwrite the stage, before its warp's arrivals hand it back
                fence_proxy_async_smem();
                __syncwarp();
                if (lane < CM) mbar_arrive_cluster(&empty[stage], lane);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            if (ep.stats_out != nullptr) {
                // (sum, M2 about the slice mean) of each 128-column slice of the new rows: the four threads of a quad share a row
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int half = 0; half < NSLICE; ++half) {
                        float s = csum[h][half];
                        s += __shfl_xor_sync(0xffffffff, s, 1);
                        s += __shfl_xor_sync(0xffffffff, s, 2);
                        const float mu = s * (1.0f / 128.0f);
                        float m2 = 0.f;
#pragma unroll
                        for (int j = 16 * half; j < 16 * half + 16; ++j) {
                            const float d0 = acc[4 * j + 2 * h] - mu, d1 = acc[4 * j + 2 * h + 1] - mu;
                            m2 = fmaf(d0, d0, fmaf(d1, d1, m2));
                        }
                        m2 += __shfl_xor_sync(0xffffffff, m2, 1);
                        m2 += __shfl_xor_sync(0xffffffff, m2, 2);
                        const int row = r0 + 8 * h;
                        if ((lane & 3) == 0 && row < M)
                            ep.stats_out[static_cast<size_t>(row) * (N / 128) + n_blk * NSLICE + half] = make_float2(s, m2);
                    }
                }
            }
        }
    }
    if constexpr (tma_store_epi(EPI))
        if ((threadIdx.x & 127) == 0) tma_store_wait<0>();  // the stores have read the staging boxes and written the output
    cluster_sync();  // the peer's consumers have made their last arrival on this CTA's barriers
}

}  // namespace gemm

// Clusters of this instantiation that fit on the GPU at once (cudaOccupancyMaxActiveClusters at set-up; the least over the
// devices set up).  Not assumed to be SM count / CM: a cluster must sit within one GPC, and GPCs differ in size.
template <int EPI, int BN, int PARTS>
static int& max_clusters() {
    static int n = 0;
    return n;
}

// Every gemm_kernel<EPI, BN, PARTS> the launchers can select, each set up at init and launched from this one list.  A launch
// selects BN = 256 when N % 256 == 0, else 128, and PARTS = e.parts_in with statistics, else 6 (not read), and is refused with
// cudaErrorInvalidValue when that instantiation is not listed.  Eight partials (bge-large's 1024-wide LayerNorm) exist for BN =
// 256 and every epilogue but quick-GELU: every bge-large N is a multiple of 256.  Four partials (the CLIP text tower's 512-wide
// LayerNorm, folded into QKV and the quick-GELU FFN1) exist for BN = 256 and EPI 0 / 3 only; its residual epilogues take no
// statistics (pre-LN).  Three partials re-applied by the residual epilogue mean N = 384, never a multiple of 256: no
// <RES_SPLIT, 256, 3>.
template <int EPI, int BN, int PARTS>
struct Inst {
    static constexpr int epi = EPI, bn = BN, parts = PARTS;
};
constexpr std::tuple<
    Inst<EPI_BIAS_F16, 256, 6>, Inst<EPI_BIAS_F16, 256, 3>, Inst<EPI_BIAS_F16, 128, 6>, Inst<EPI_BIAS_F16, 128, 3>,
    Inst<EPI_BIAS_F16, 256, 4>, Inst<EPI_BIAS_F16, 256, 8>,
    Inst<EPI_BIAS_GELU_F16, 256, 6>, Inst<EPI_BIAS_GELU_F16, 256, 3>, Inst<EPI_BIAS_GELU_F16, 128, 6>, Inst<EPI_BIAS_GELU_F16, 128, 3>,
    Inst<EPI_BIAS_GELU_F16, 256, 8>,
    Inst<EPI_BIAS_QGELU_F16, 256, 6>, Inst<EPI_BIAS_QGELU_F16, 256, 3>, Inst<EPI_BIAS_QGELU_F16, 128, 6>, Inst<EPI_BIAS_QGELU_F16, 128, 3>,
    Inst<EPI_BIAS_QGELU_F16, 256, 4>,
    Inst<EPI_BIAS_RES_SPLIT, 256, 6>, Inst<EPI_BIAS_RES_SPLIT, 128, 6>, Inst<EPI_BIAS_RES_SPLIT, 128, 3>, Inst<EPI_BIAS_RES_SPLIT, 256, 8>,
    Inst<EPI_SPLADE_MAX, 256, 6>, Inst<EPI_SPLADE_MAX, 256, 3>, Inst<EPI_SPLADE_MAX, 256, 8>,
    Inst<EPI_ROPE_F16, 256, 6>,
    Inst<EPI_SWIGLU_F16, 256, 6>>
    INSTANTIATIONS{};

template <int EPI, int BN, int PARTS>
static cudaError_t setup(Inst<EPI, BN, PARTS>) {
    auto kernel = gemm::gemm_kernel<EPI, BN, PARTS>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, gemm::smem_bytes<EPI, BN>());
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};  // the cluster shape comes from the kernel's __cluster_dims__
    cfg.gridDim = dim3(gemm::CM);
    cfg.blockDim = dim3(gemm::NUM_THREADS);
    cfg.dynamicSmemBytes = gemm::smem_bytes<EPI, BN>();
    int n = 0;
    if ((e = cudaOccupancyMaxActiveClusters(&n, kernel, &cfg)) != cudaSuccess) return e;
    if (n < 1) return cudaErrorInvalidConfiguration;
    int& m = max_clusters<EPI, BN, PARTS>();
    m = m == 0 ? n : std::min(m, n);
    return cudaSuccess;
}

cudaError_t gemm_init_device() {
    cudaError_t e = cudaSuccess;
    std::apply([&](auto... inst) { (((e = setup(inst)) == cudaSuccess) && ...); }, INSTANTIATIONS);
    return e;
}

template <int EPI, int BN, int PARTS>
static cudaError_t launch_one(Inst<EPI, BN, PARTS>, const CUtensorMap& ta, const CUtensorMap& tb, __half* out, __half* out_lo,
                              const GemmEpi& e, int M, int N, int K, int sm_count, cudaStream_t stream, int* ctas, const SpladeEpi& sp,
                              const RopeEpi& rp, const ResEpi& res, const OutEpi& oe) {
    const int pairs = ((M + gemm::CM * gemm::BM - 1) / (gemm::CM * gemm::BM)) * (N / BN);
    int clusters = std::min({pairs, sm_count / gemm::CM, max_clusters<EPI, BN, PARTS>()});
    if (clusters < 1) clusters = 1;
    if (ctas) *ctas = clusters * gemm::CM;
    return launch_pdl(gemm::gemm_kernel<EPI, BN, PARTS>, dim3(clusters * gemm::CM), dim3(gemm::NUM_THREADS), gemm::smem_bytes<EPI, BN>(),
                      stream, ta, tb, e, out, out_lo, M, N, K, sp, rp, res, oe);
}

// launches the listed instantiation that epilogue `epi` selects for these operands (see INSTANTIATIONS)
static cudaError_t launch_listed(int epi, const CUtensorMap& ta, const CUtensorMap& tb, __half* out, __half* out_lo, const GemmEpi& e, int M,
                                 int N, int K, int sm_count, cudaStream_t stream, int* ctas, const SpladeEpi& sp = SpladeEpi{},
                                 const RopeEpi& rp = RopeEpi{}, const ResEpi& res = ResEpi{}, const OutEpi& oe = OutEpi{}) {
    const int bn = N % 256 == 0 ? 256 : 128, parts = e.stats_in != nullptr ? e.parts_in : 6;
    cudaError_t r = cudaErrorInvalidValue;
    std::apply([&](auto... inst) {
        ((inst.epi == epi && inst.bn == bn && inst.parts == parts && (r = launch_one(inst, ta, tb, out, out_lo, e, M, N, K, sm_count, stream,
                                                                                  ctas, sp, rp, res, oe), true)) || ...);
    }, INSTANTIATIONS);
    return r;
}

cudaError_t launch_gemm(int epi, const CUtensorMap& ta, const CUtensorMap& tb, __half* out, __half* out_lo, const ResEpi* res,
                        const OutEpi* oe, const GemmEpi& e, int M, int N, int K, int sm_count, cudaStream_t stream, int* ctas) {
    if (N % 128 != 0 || K % gemm::BK != 0 || M <= 0 || e.bias == nullptr || out == nullptr || sm_count < 1) return cudaErrorInvalidValue;
    // the statistics describe the LayerNorm'd row: K wide for a folded LayerNorm, N wide for the residual re-apply
    const bool resid = epi == EPI_BIAS_RES_SPLIT;
    if (e.stats_in != nullptr && e.parts_in * 128 != (resid ? N : K)) return cudaErrorInvalidValue;
    if (gemm::tma_store_epi(epi)) {
        if (oe == nullptr) return cudaErrorInvalidValue;
        return launch_listed(epi, ta, tb, out, nullptr, e, M, N, K, sm_count, stream, ctas, SpladeEpi{}, RopeEpi{}, ResEpi{}, *oe);
    }
    if (!resid || out_lo == nullptr || res == nullptr || (e.stats_in != nullptr && (e.ln_gamma == nullptr || e.ln_beta == nullptr)))
        return cudaErrorInvalidValue;
    if (e.stats_out != nullptr && e.stats_out == e.stats_in) return cudaErrorInvalidValue;
    return launch_listed(epi, ta, tb, out, out_lo, e, M, N, K, sm_count, stream, ctas, SpladeEpi{}, RopeEpi{}, *res);
}

cudaError_t launch_gemm_splade(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpi& e, const SpladeEpi& sp, int M, int N, int K,
                               int sm_count, cudaStream_t stream, int* ctas) {
    if (N % 256 != 0 || K % gemm::BK != 0 || M <= 0 || sm_count < 1 || e.bias == nullptr || e.stats_in == nullptr || e.parts_in * 128 != K)
        return cudaErrorInvalidValue;
    if (sp.lens == nullptr || sp.vmax == nullptr || sp.S < 64 || sp.S % 64 != 0 || M % sp.S != 0 || sp.vocab < 1 || sp.vocab > N)
        return cudaErrorInvalidValue;
    return launch_listed(EPI_SPLADE_MAX, ta, tb, nullptr, nullptr, e, M, N, K, sm_count, stream, ctas, sp);
}

cudaError_t launch_gemm_rope(const CUtensorMap& ta, const CUtensorMap& tb, __half* out, const GemmEpi& e, const RopeEpi& rp, int M, int N,
                             int K, int sm_count, cudaStream_t stream, int* ctas) {
    if (N % 256 != 0 || K != 768 || M <= 0 || sm_count < 1 || out == nullptr || e.bias == nullptr) return cudaErrorInvalidValue;
    if (rp.table == nullptr || rp.S < 64 || rp.S % 64 != 0 || rp.rot_cols < 0 || rp.rot_cols % 256 != 0 || rp.rot_cols > N) return cudaErrorInvalidValue;
    return launch_listed(EPI_ROPE_F16, ta, tb, out, nullptr, e, M, N, K, sm_count, stream, ctas, SpladeEpi{}, rp);
}

cudaError_t launch_gemm_swiglu(const CUtensorMap& ta, const CUtensorMap& tb, __half* out, const GemmEpi& e, int M, int N, int K, int sm_count,
                               cudaStream_t stream, int* ctas) {
    if (N % 256 != 0 || K != 768 || M <= 0 || sm_count < 1 || out == nullptr || e.bias == nullptr) return cudaErrorInvalidValue;
    return launch_listed(EPI_SWIGLU_F16, ta, tb, out, nullptr, e, M, N, K, sm_count, stream, ctas);
}

}  // namespace b200
