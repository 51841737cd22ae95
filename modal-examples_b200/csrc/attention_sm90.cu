// Multi-head self-attention for S <= 512, NH heads of d: 12 of 64 (bge-base), 12 of 32 (bge-small), 16 of 64 (bge-large) or,
// causal, 8 of 64 (CLIP's text tower), on wgmma (sm_90a): persistent CTAs.  The kernel is a template on (d, NH, CAUSAL); the
// comments below give the d = 64 figures, d = 32 differences follow.  NH only sets the unit decode and the column offsets of K
// and V.
//
// A work unit is one (item, head) -- or, for batches with fewer units than SMs, one (item, head, query tile).  Each CTA walks
// the units u = blockIdx.x, blockIdx.x + gridDim.x, ...  For the unit in hand one thread TMA-loads the head's K and V
// (<= 512 x 64 fp16 each, up to four 128-key tiles, one mbarrier per tile) and the unit's 128-row query tiles (double
// buffered) into 128B-swizzled shared memory; everything is issued up front, so the first sub-block's MMAs start as soon as
// its own tile has landed.
//
// Two warpgroups; warpgroup c takes query rows 64c .. 64c+63 of every tile and walks the keys in 64-key sub-blocks:
//   S   = Q . K_c^T      four wgmma.m64n64k16 (Q and K from shared memory, both K-major), fp32 in registers;
//   online softmax       row max over the quad of threads that share a row, P = exp2((S - m) k) with k = log2(e) / 8, the
//                        output accumulator and the partial row sum rescaled by exp2((m_old - m) k);
//   O  += P . V_c        four wgmma.m64n64k16 with A = P (fp16) straight from the registers -- the S accumulator fragment
//                        is already the A-operand fragment of the same rows -- and B = V_c (MN-major) from shared memory.
// The tile's output ctx = O / l is staged in the tile's own (now idle) query buffer and leaves with one TMA store.
//
// d = 32: a row of Q, K or V is 64 bytes, so every tile is 64B-swizzled (TMA box {32, 128, 1}, 8 KB per 128 rows); S = Q . K^T
// is two k-steps of m64n64k16 and O += P . V four m64n32k16 (16 fp32 O registers per thread); the softmax scale is 1/sqrt(32).
//
// Keys >= len are masked to -inf before the max (exactly P = 0, matching HF's additive -inf mask); sub-blocks wholly past
// len are skipped.
//
// CAUSAL (CLIPTextTransformer's causal mask): key k is also masked for query row q when k > q, at the same place as the len
// mask.  The rows of warpgroup wg in query tile t are (t0 + t) 128 + 64 wg ... + 63, so its sub-block 2 (t0 + t) + wg is the
// diagonal one (masked per row) and every later sub-block is wholly masked: the warpgroup stops there.  Running a wholly
// masked sub-block would change nothing bitwise -- the row max stays, alpha = exp2(0) = 1, p = exp2(-inf) = 0, O and l get
// exact zeros added -- so skipping it keeps the output independent of batch, bucket, CTA and query-tile split.  A unit loads
// only the K / V tiles its last query tile reaches (warpgroup 1 of that tile waits on every one of them).  Sub-block 0 holds
// key 0 for every row, so no row is ever fully masked and padding rows stay finite.  Every query tile is computed the same way whether the item travels as one unit or split by query tile,
// alone or in any batch, on any CTA, so an item's embedding is bit-identical in any batch (tests: scheduler / size-independent
// properties).
//
// Restates BertSelfAttention.forward (HF modeling_bert.py:143-207) for the TEI /embed path the
// reference calls at 06_gpu_and_ml/embeddings/text_embeddings_inference.py:100.
#include <tuple>

#include "kernels.h"
#include "ptx.cuh"

namespace b200 {
namespace attn {

constexpr int QT = 128;      // query rows per tile
constexpr int KB = 128;      // keys per K/V smem tile (TMA box)
constexpr int SB = 64;       // keys per sub-block
constexpr int MAX_KB = 4;    // S <= 512
constexpr int NUM_THREADS = 256;

// Shared-memory layout of the head-dim-D kernel: rows of RB = 2D bytes (128 or 64), each tile 128 rows.
template <int D>
struct Layout {
    static constexpr int RB = 2 * D;                                // bytes per row
    static constexpr int TILE_BYTES = 128 * RB;                     // 16 KB (d = 64) / 8 KB (d = 32)
    static constexpr int OFF_Q = 0;                                 // 2 tiles (double buffered across tiles), also the output staging
    static constexpr int OFF_K = OFF_Q + 2 * TILE_BYTES;            // MAX_KB tiles
    static constexpr int OFF_V = OFF_K + MAX_KB * TILE_BYTES;       // MAX_KB tiles
    static constexpr int OFF_BAR = OFF_V + MAX_KB * TILE_BYTES;
    static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
    static_assert(SMEM_BYTES <= 232448, "shared memory");
};

// softmax_scale * log2(e) with softmax_scale = 1/sqrt(D)
template <int D>
constexpr float scale_log2e() { return (D == 64 ? 0.125f : 0.17677669529663687f) * 1.4426950408889634f; }

// descriptor of a K-major (Q, K) or MN-major (V) operand tile of the head-dim-D layout
template <int D>
__device__ __forceinline__ uint64_t make_desc(uint32_t addr) {
    if constexpr (D == 64) return make_sw128_desc(addr);
    else return make_sw64_desc(addr);
}

struct Unit {
    int b, h, t0, nq;  // item, head, first query tile, query tiles
    int len, nsb, nkb; // valid keys, 64-key sub-blocks, 128-key K/V tiles
};

template <int NH, bool CAUSAL>
__device__ __forceinline__ Unit decode_unit(int u, int nq_all, int split, const int32_t* __restrict__ lens, int S) {
    Unit U;
    int unit = u;
    U.t0 = 0;
    if (split) {
        U.t0 = unit % nq_all;
        unit /= nq_all;
    }
    U.b = unit / NH;
    U.h = unit % NH;
    int len = __ldg(lens + U.b);
    len = len < 1 ? 1 : (len > S ? S : len);
    U.len = len;
    U.nq = split ? 1 : nq_all;
    U.nsb = (len + SB - 1) / SB;
    if constexpr (CAUSAL) U.nsb = min(U.nsb, 2 * (U.t0 + U.nq));  // keys past the unit's last query row are never needed
    U.nkb = (U.nsb + 1) / 2;
    return U;
}

template <int D, int NH, bool CAUSAL = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tctx,
                 const int32_t* __restrict__ lens, int S, int split, int n_units) {
    using L = Layout<D>;
    constexpr int RB = L::RB, TILE_BYTES = L::TILE_BYTES, OFF_Q = L::OFF_Q, OFF_K = L::OFF_K, OFF_V = L::OFF_V, OFF_BAR = L::OFF_BAR;
    constexpr int HID = NH * D;        // ctx width; qkv rows are 3 HID wide (Q | K | V)
    constexpr int NO = D / 2;          // O accumulators per thread
    constexpr float kScaleLog2e = scale_log2e<D>();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* kv_full = bars;          // [MAX_KB]  K tile j and V tile j of the unit have landed
    uint64_t* q_full = bars + MAX_KB;  // [2]

    griddep_launch_dependents();
    const int lane = lane_id();
    const int wg = threadIdx.x >> 7;          // which 64 query rows of a tile
    const int w4 = (threadIdx.x >> 5) & 3;    // warp within the warpgroup: rows 16 w4 .. 16 w4 + 15
    const int nq_all = (S + QT - 1) / QT;
    const bool loader = threadIdx.x == 0;

    if (loader) {
        prefetch_tmap(&tq);
        prefetch_tmap(&tctx);
        for (int i = 0; i < MAX_KB; ++i) mbar_init(&kv_full[i], 1);
        for (int i = 0; i < 2; ++i) mbar_init(&q_full[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    griddep_wait();  // the prologue above overlapped the previous kernel's tail; nothing it wrote (qkv, lens) has been read yet

    // this thread's rows of a tile (first and +8) and their 16-byte chunk in a swizzled row: dims 8j .. 8j+7 of row r
    // sit in chunk j ^ (r & 7) (128-byte rows) or j ^ ((r >> 1) & 3) (64-byte rows)
    const int rr = wg * 64 + w4 * 16 + (lane >> 2);
    const uint32_t cq = 4 * (lane & 3);  // byte offset of this thread's two dims inside a chunk
    uint32_t kv_par = 0;                 // bit j: parity of the number of loads of K/V tile j so far
    uint32_t gt = 0;                     // the CTA's running query-tile index
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const Unit U = decode_unit<NH, CAUSAL>(u, nq_all, split, lens, S);
        auto load_q = [&](uint32_t g, int t) {
            mbar_arrive_expect_tx(&q_full[g & 1], TILE_BYTES);
            tma_load_3d(smem + OFF_Q + (g & 1) * TILE_BYTES, &tq, &q_full[g & 1], U.h * D, (U.t0 + t) * QT, U.b);
        };
        if (loader) {
            load_q(gt, 0);
            for (int j = 0; j < U.nkb; ++j) {
                mbar_arrive_expect_tx(&kv_full[j], 2 * TILE_BYTES);
                tma_load_3d(smem + OFF_K + j * TILE_BYTES, &tq, &kv_full[j], HID + U.h * D, j * KB, U.b);
                tma_load_3d(smem + OFF_V + j * TILE_BYTES, &tq, &kv_full[j], 2 * HID + U.h * D, j * KB, U.b);
            }
            if (U.nq > 1) load_q(gt + 1, 1);
        }
        for (int t = 0; t < U.nq; ++t) {
            const uint32_t g = gt + t;
            const uint32_t q_buf = smem_u32(smem + OFF_Q + (g & 1) * TILE_BYTES);
            mbar_wait(&q_full[g & 1], (g >> 1) & 1);
            float o[NO];
#pragma unroll
            for (int i = 0; i < NO; ++i) o[i] = 0.f;
            float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
            const uint32_t q_addr = q_buf + wg * (64 * RB);
            int nsb = U.nsb;
            if constexpr (CAUSAL) nsb = min(nsb, 2 * (U.t0 + t) + wg + 1);  // up to this warpgroup's diagonal sub-block
#pragma unroll 1
            for (int sb = 0; sb < nsb; ++sb) {
                if ((sb & 1) == 0) mbar_wait(&kv_full[sb >> 1], (kv_par >> (sb >> 1)) & 1);
                const uint32_t k_addr = smem_u32(smem + OFF_K) + sb * (SB * RB);
                float s[32];
                wgmma_fence();
                fence_operands(s);
#pragma unroll
                for (int k = 0; k < D / 16; ++k)
                    wgmma_m64n64k16_ss(s, make_desc<D>(q_addr + k * 32), make_desc<D>(k_addr + k * 32), k != 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_operands(s);
                const int valid = U.len - sb * SB;  // keys [0, valid) of this sub-block are real (>= 1)
                if (valid < SB) {
#pragma unroll
                    for (int i = 0; i < 32; ++i)
                        if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= valid) s[i] = -INFINITY;
                }
                if constexpr (CAUSAL) {
                    if (sb == 2 * (U.t0 + t) + wg) {  // diagonal: key column c > row r of the warpgroup's 64 is in the future
#pragma unroll
                        for (int i = 0; i < 32; ++i)
                            if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) > w4 * 16 + (lane >> 2) + 8 * ((i >> 1) & 1)) s[i] = -INFINITY;
                    }
                }
                uint32_t pa[4][4];  // P as the A fragments of the four 16-key steps
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float mx = -INFINITY;
#pragma unroll
                    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffff, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffff, mx, 2));
                    const float m_new = fmaxf(m_run[h], mx);
                    const float alpha = ex2_approx((m_run[h] - m_new) * kScaleLog2e);  // 0 on the first sub-block
                    m_run[h] = m_new;
                    const float neg_ms = -m_new * kScaleLog2e;
                    float ls = 0.f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float p0 = ex2_approx(fmaf(s[4 * j + 2 * h], kScaleLog2e, neg_ms));
                        const float p1 = ex2_approx(fmaf(s[4 * j + 2 * h + 1], kScaleLog2e, neg_ms));
                        ls += p0 + p1;
                        // keys 8j .. 8j+7: k-step j/2, register 2 (j odd) + h
                        pa[j >> 1][2 * (j & 1) + h] = pack_half2(p0, p1);
                        if (j < D / 8) {  // O has D / 8 column groups
                            o[4 * j + 2 * h] *= alpha;
                            o[4 * j + 2 * h + 1] *= alpha;
                        }
                    }
                    l_run[h] = fmaf(l_run[h], alpha, ls);
                }
                const uint32_t v_addr = smem_u32(smem + OFF_V) + sb * (SB * RB);
                wgmma_fence();
                fence_operands(o);
#pragma unroll
                for (int kk = 0; kk < SB / 16; ++kk) {
                    if constexpr (D == 64) wgmma_m64n64k16_rs_mn(o, pa[kk], make_desc<D>(v_addr + kk * (16 * RB)), 1);
                    else wgmma_m64n32k16_rs_mn(o, pa[kk], make_desc<D>(v_addr + kk * (16 * RB)), 1);
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_operands(o);
            }
            // ctx = O / l, staged over this warpgroup's own rows of the tile's query buffer (its MMAs on them are complete)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float l = l_run[h];
                l += __shfl_xor_sync(0xffffffff, l, 1);
                l += __shfl_xor_sync(0xffffffff, l, 2);
                const float inv_l = 1.0f / l;
                const int r = rr + 8 * h;
                const uint32_t row = q_buf + r * RB + cq;
                const uint32_t sw = (static_cast<uint32_t>(r) * RB >> 7) & (RB / 16 - 1);  // the row's chunk swizzle
#pragma unroll
                for (int j = 0; j < D / 8; ++j)
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(row + ((static_cast<uint32_t>(j) ^ sw) << 4)),
                                 "r"(pack_half2(o[4 * j + 2 * h] * inv_l, o[4 * j + 2 * h + 1] * inv_l))
                                 : "memory");
            }
            fence_proxy_async_smem();
            __syncthreads();
            if (loader) {  // rows past S are clipped by the tensor map
                tma_store_3d(&tctx, smem + OFF_Q + (g & 1) * TILE_BYTES, U.h * D, (U.t0 + t) * QT, U.b);
                tma_store_commit();
                tma_store_wait_read<0>();  // the buffer is free again
                if (t + 2 < U.nq) load_q(g + 2, t + 2);
            }
        }
        kv_par ^= (1u << U.nkb) - 1;
        gt += U.nq;
        __syncthreads();  // K / V are reloaded for the next unit only once every warpgroup is done with them
    }
    if (loader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores complete before exit
}


// ------------------------------------------------------------------------------------------------------------------------
// Streaming K/V attention, any S up to 8192 (a multiple of 64), 12 heads of 64 (nomic-bert): the K and V of a head no longer
// fit in shared memory, so they stream through a ring of NSTAGE 128-key stages (K and V 16 KB each, one `full` mbarrier with
// the stage's tx-count and one `empty` mbarrier taking an arrival from each of the 8 consumer warps).
//
// A unit is one (item b, head h, 128-row query tile t), numbered ((b NH + h) nq + t): the query tiles of a head are adjacent,
// so the CTAs that run together read that head's K / V from L2 rather than HBM.  Persistent CTAs walk u = blockIdx.x,
// blockIdx.x + gridDim.x, ...  Three warpgroups:
//   warpgroup 0 (setmaxnreg 40): one thread TMA-loads the unit's Q tile (double buffered: q_full / q_empty) and its
//       ceil(len / 128) K / V tiles into the ring -- never the padding past the item's length -- and runs ahead across units;
//   warpgroups 1-2 (setmaxnreg 232): consumer c takes query rows 64c .. 64c + 63 of the tile and walks the keys in 64-key
//       sub-blocks exactly as attention_kernel<64, NH> does: the same wgmma sequence, -inf mask past len, online softmax with
//       ex2.approx, rescale and P . V from registers, in the same key order.  At S <= 512 its ctx is therefore bit-identical
//       to attention_kernel's on the same qkv, and an item's ctx does not depend on the batch, the bucket, the grid or the CTA.
//       A consumer frees a stage after its second sub-block (or the unit's last), the Q buffer after the unit's last
//       sub-block, and stores ctx = O / l straight from its registers (rows past S are not stored).
// Shared memory: Q 2 x 16 KB + NSTAGE x 32 KB + barriers = 165 120 bytes with NSTAGE = 4.
namespace stream {
constexpr int NSTAGE = 4;
constexpr int NUM_THREADS = 384;
constexpr int TILE_BYTES = 128 * 128;               // 128 rows of 64 fp16, 128B-swizzled
constexpr int OFF_Q = 0;                            // 2 tiles
constexpr int OFF_KV = 2 * TILE_BYTES;              // stage s: K at OFF_KV + 2 s TILE_BYTES, V one tile later
constexpr int OFF_BAR = OFF_KV + NSTAGE * 2 * TILE_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "shared memory");
constexpr int MAX_S = 8192;
}  // namespace stream

template <int D, int NH>
__global__ void __launch_bounds__(stream::NUM_THREADS, 1)
attention_stream_kernel(const __grid_constant__ CUtensorMap tq, __half* __restrict__ ctx, const int32_t* __restrict__ lens, int S,
                        int n_units) {
    static_assert(D == 64, "128-byte rows");
    using namespace stream;
    constexpr int RB = 2 * D;
    constexpr int HID = NH * D;
    constexpr int NO = D / 2;
    constexpr float kScaleLog2e = scale_log2e<D>();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* kv_full = bars;                 // [NSTAGE]
    uint64_t* kv_empty = bars + NSTAGE;       // [NSTAGE]
    uint64_t* q_full = bars + 2 * NSTAGE;     // [2]
    uint64_t* q_empty = bars + 2 * NSTAGE + 2;  // [2]

    griddep_launch_dependents();
    const int warp = __shfl_sync(0xffffffff, threadIdx.x >> 5, 0);
    const int lane = lane_id();
    const int nq = (S + QT - 1) / QT;
    if (threadIdx.x == 0) {
        prefetch_tmap(&tq);
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(&kv_full[s], 1);
            mbar_init(&kv_empty[s], 8);  // the 8 consumer warps
        }
        for (int i = 0; i < 2; ++i) {
            mbar_init(&q_full[i], 1);
            mbar_init(&q_empty[i], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();
    griddep_wait();  // the prologue above overlapped the previous kernel's tail; nothing it wrote (qkv, lens) has been read yet

    // unit u -> item, head, query tile and the item's valid keys (clamped to [1, S]), its 64-key sub-blocks
    auto decode = [&](int u, int& b, int& h, int& t, int& len, int& nsb) {
        t = u % nq;
        const int bh = u / nq;
        h = bh % NH;
        b = bh / NH;
        len = __ldg(lens + b);
        len = len < 1 ? 1 : (len > S ? S : len);
        nsb = (len + SB - 1) / SB;
    };

    if (warp < 4) {
        // -------------------------------------------------------------------- TMA producer
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            int stage = 0;
            uint32_t phase = 0, g = 0;
            for (int u = blockIdx.x; u < n_units; u += gridDim.x, ++g) {
                int b, h, t, len, nsb;
                decode(u, b, h, t, len, nsb);
                mbar_wait(&q_empty[g & 1], ((g >> 1) & 1) ^ 1);  // the unit two before this one has finished with the buffer
                mbar_arrive_expect_tx(&q_full[g & 1], TILE_BYTES);
                tma_load_3d(smem + OFF_Q + (g & 1) * TILE_BYTES, &tq, &q_full[g & 1], h * D, t * QT, b);
                for (int j = 0; j < (nsb + 1) / 2; ++j) {
                    mbar_wait(&kv_empty[stage], phase ^ 1);
                    uint8_t* st = smem + OFF_KV + stage * 2 * TILE_BYTES;
                    mbar_arrive_expect_tx(&kv_full[stage], 2 * TILE_BYTES);  // keys past S are zero-filled and still counted
                    tma_load_3d(st, &tq, &kv_full[stage], HID + h * D, j * KB, b);
                    tma_load_3d(st + TILE_BYTES, &tq, &kv_full[stage], 2 * HID + h * D, j * KB, b);
                    if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
                }
            }
        }
        __syncwarp();
        return;
    }

    // ------------------------------------------------------------------------ consumers
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;  // which 64 query rows of a tile
    const int w4 = warp & 3;         // rows 16 w4 .. 16 w4 + 15 of them
    int stage = 0;
    uint32_t phase = 0, g = 0;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x, ++g) {
        int b, h, t, len, nsb;
        decode(u, b, h, t, len, nsb);
        mbar_wait(&q_full[g & 1], (g >> 1) & 1);
        float o[NO];
#pragma unroll
        for (int i = 0; i < NO; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        const uint32_t q_addr = smem_u32(smem + OFF_Q + (g & 1) * TILE_BYTES) + wg * (64 * RB);
#pragma unroll 1
        for (int sb = 0; sb < nsb; ++sb) {
            if ((sb & 1) == 0) mbar_wait(&kv_full[stage], phase);
            const uint32_t k_addr = smem_u32(smem + OFF_KV + stage * 2 * TILE_BYTES) + (sb & 1) * (SB * RB);
            float s[32];
            wgmma_fence();
            fence_operands(s);
#pragma unroll
            for (int k = 0; k < D / 16; ++k)
                wgmma_m64n64k16_ss(s, make_desc<D>(q_addr + k * 32), make_desc<D>(k_addr + k * 32), k != 0);
            wgmma_commit();
            wgmma_wait<0>();
            fence_operands(s);
            const int valid = len - sb * SB;  // keys [0, valid) of this sub-block are real (>= 1)
            if (valid < SB) {
#pragma unroll
                for (int i = 0; i < 32; ++i)
                    if (8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= valid) s[i] = -INFINITY;
            }
            uint32_t pa[4][4];  // P as the A fragments of the four 16-key steps
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                float mx = -INFINITY;
#pragma unroll
                for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * hf], s[4 * j + 2 * hf + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffff, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffff, mx, 2));
                const float m_new = fmaxf(m_run[hf], mx);
                const float alpha = ex2_approx((m_run[hf] - m_new) * kScaleLog2e);  // 0 on the first sub-block
                m_run[hf] = m_new;
                const float neg_ms = -m_new * kScaleLog2e;
                float ls = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float p0 = ex2_approx(fmaf(s[4 * j + 2 * hf], kScaleLog2e, neg_ms));
                    const float p1 = ex2_approx(fmaf(s[4 * j + 2 * hf + 1], kScaleLog2e, neg_ms));
                    ls += p0 + p1;
                    pa[j >> 1][2 * (j & 1) + hf] = pack_half2(p0, p1);
                    o[4 * j + 2 * hf] *= alpha;
                    o[4 * j + 2 * hf + 1] *= alpha;
                }
                l_run[hf] = fmaf(l_run[hf], alpha, ls);
            }
            const uint32_t v_addr = smem_u32(smem + OFF_KV + stage * 2 * TILE_BYTES + TILE_BYTES) + (sb & 1) * (SB * RB);
            wgmma_fence();
            fence_operands(o);
#pragma unroll
            for (int kk = 0; kk < SB / 16; ++kk) wgmma_m64n64k16_rs_mn(o, pa[kk], make_desc<D>(v_addr + kk * (16 * RB)), 1);
            wgmma_commit();
            wgmma_wait<0>();
            fence_operands(o);
            if ((sb & 1) || sb == nsb - 1) {  // the stage's last sub-block: hand it back to the producer
                if (lane == 0) mbar_arrive(&kv_empty[stage]);
                if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
            }
        }
        if (lane == 0) mbar_arrive(&q_empty[g & 1]);  // this warp's last MMA on the Q tile has completed
        // ctx = O / l, straight from the registers: this thread's rows r and r + 8 of the tile, dims 8j + 2 (lane % 4) + {0, 1}
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            float l = l_run[hf];
            l += __shfl_xor_sync(0xffffffff, l, 1);
            l += __shfl_xor_sync(0xffffffff, l, 2);
            const float inv_l = 1.0f / l;
            const int r = t * QT + wg * 64 + w4 * 16 + (lane >> 2) + 8 * hf;
            if (r < S) {
                __half* row = ctx + (static_cast<size_t>(b) * S + r) * HID + h * D + 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < D / 8; ++j)
                    *reinterpret_cast<uint32_t*>(row + 8 * j) = pack_half2(o[4 * j + 2 * hf] * inv_l, o[4 * j + 2 * hf + 1] * inv_l);
            }
        }
    }
}

}  // namespace attn

// Every attention_kernel<D, NH, CAUSAL> launch_attention can select, each set up at init and launched from this one list:
// (head_dim, heads) = (64, 12) bge-base and ViT, (32, 12) bge-small, (64, 16) bge-large, and (64, 8) causal, the CLIP text tower.
template <int D, int NH, bool CAUSAL>
struct Inst {
    static constexpr int d = D, nh = NH;
    static constexpr bool causal = CAUSAL;
};
constexpr std::tuple<Inst<64, 12, false>, Inst<32, 12, false>, Inst<64, 16, false>, Inst<64, 8, true>> INSTANTIATIONS{};

template <int D, int NH, bool CAUSAL>
static cudaError_t setup(Inst<D, NH, CAUSAL>) {
    return cudaFuncSetAttribute(attn::attention_kernel<D, NH, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn::Layout<D>::SMEM_BYTES);
}

template <int D, int NH, bool CAUSAL>
static cudaError_t launch_one(Inst<D, NH, CAUSAL>, const CUtensorMap& tq, const CUtensorMap& tctx, const int32_t* lens, int B, int S,
                              int sm_count, cudaStream_t stream) {
    // fewer (item, head) units than SMs: split them by query tile (K and V are then loaded once per tile, but a single item
    // spreads over 4 NH SMs instead of NH)
    const int nq = (S + attn::QT - 1) / attn::QT;
    const int split = (B * NH < sm_count && nq > 1) ? 1 : 0;
    const int n_units = B * NH * (split ? nq : 1);
    const int grid = n_units < sm_count ? n_units : sm_count;
    return launch_pdl(attn::attention_kernel<D, NH, CAUSAL>, dim3(grid), dim3(attn::NUM_THREADS), attn::Layout<D>::SMEM_BYTES, stream, tq, tctx, lens,
                      S, split, n_units);
}

cudaError_t attention_init_device() {
    cudaError_t e = cudaSuccess;
    std::apply([&](auto... inst) { (((e = setup(inst)) == cudaSuccess) && ...); }, INSTANTIATIONS);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(attn::attention_stream_kernel<64, 12>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn::stream::SMEM_BYTES);
}

cudaError_t launch_attention(const CUtensorMap& tq, const CUtensorMap& tctx, const int32_t* lens, int B, int S, int sm_count,
                             cudaStream_t stream, int head_dim, int heads, bool causal) {
    if (S < 1 || S > attn::MAX_KB * attn::KB || B < 1 || sm_count < 1) return cudaErrorInvalidValue;
    cudaError_t r = cudaErrorInvalidValue;
    std::apply([&](auto... inst) {
        ((inst.d == head_dim && inst.nh == heads && inst.causal == causal && (r = launch_one(inst, tq, tctx, lens, B, S, sm_count, stream), true)) ||
         ...);
    }, INSTANTIATIONS);
    return r;
}

cudaError_t launch_attention_stream(const CUtensorMap& tq, __half* ctx, const int32_t* lens, int B, int S, int sm_count, cudaStream_t stream) {
    if (S < 64 || S % 64 != 0 || S > attn::stream::MAX_S || B < 1 || sm_count < 1 || ctx == nullptr || lens == nullptr) return cudaErrorInvalidValue;
    const int n_units = B * 12 * ((S + attn::QT - 1) / attn::QT);
    const int grid = n_units < sm_count ? n_units : sm_count;
    return launch_pdl(attn::attention_stream_kernel<64, 12>, dim3(grid), dim3(attn::stream::NUM_THREADS), attn::stream::SMEM_BYTES, stream, tq,
                      ctx, lens, S, n_units);
}

}  // namespace b200
