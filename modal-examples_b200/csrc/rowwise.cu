// HBM-bound row-wise kernels (sm_90a): embedding gather into the split residual stream, CLS or mean pooling + final LayerNorm +
// L2 normalise with the store aimed at the root GPU's gather buffer, the root-side scatter of token ids into (peer) shard
// inputs, and the load-time weight preparation (fp32 -> fp16, LayerNorm gamma folded into weight columns).
//
// Row kernels: one warp per row (768 wide, or 384 / 1024 for bge-small's / bge-large's embed / pool / LayerNorm, 512 for the CLIP
// text tower's embed and pool), 128-bit accesses, statistics
// by warp shuffle in fp32, two-pass variance on register-resident data (no E[x^2]-E[x]^2 cancellation).
//
// The residual stream is stored PRE-LayerNorm as y = hi + lo (fp16 + fp16) together with one (sum, M2) partial per 128
// columns of each row; there is no LayerNorm kernel in the product path -- the consuming GEMM folds it into its epilogue (kernels.h).
//
// Restates BertEmbeddings.forward (HF modeling_bert.py:72-111), the LayerNorm halves of
// BertSelfOutput :287-298 / BertOutput :345-356, and sentence-transformers' CLS pooling + Normalize
// (reference 06_gpu_and_ml/gpu_snapshot.py:58, `normalize_embeddings=True`).
#include <climits>

#include "kernels.h"
#include "ptx.cuh"

namespace b200 {
namespace rw {

// Row width W: float4 i of lane l holds columns [128 i + 4 l, +4), i < W / 128 -- so float4 i of every lane covers exactly the
// i-th 128-column statistic slice.  The ViT kernels are 768 wide only.
constexpr int H = HIDDEN;  // 768
template <int W>
struct Row {
    static_assert(W == 768 || W == 384 || W == 1024 || W == 512, "row width");
    static constexpr int V4 = W / 128;  // float4 per lane: 6, 3, 8 or 4
};
constexpr int V4 = Row<H>::V4;
constexpr int WARPS_PER_BLOCK = 8;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffff, v, o);
    return v;
}

// normalise the 4 W / 128 register-resident values of this lane in place; returns (mean, rstd) of the row
template <int W = H>
__device__ __forceinline__ float2 ln_inplace(float4 (&x)[Row<W>::V4], const float* __restrict__ gamma,
                                             const float* __restrict__ beta, float eps, int lane) {
    constexpr int V4 = Row<W>::V4;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) s += (x[i].x + x[i].y) + (x[i].z + x[i].w);
    // __fmul_rn: the rounded mean itself is subtracted.  A plain product would be contracted into the subtractions below
    // (fma(-s, 1/768, x)), which see the unrounded s * fl(1/768): a constant row then centres to -x * 2^-25 instead of 0,
    // and rstd = eps^-1/2 blows that up into a unit vector where LayerNorm + F.normalize give zeros.
    const float mean = __fmul_rn(warp_sum(s), 1.0f / W);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        x[i].x -= mean; x[i].y -= mean; x[i].z -= mean; x[i].w -= mean;
        q += (x[i].x * x[i].x + x[i].y * x[i].y) + (x[i].z * x[i].z + x[i].w * x[i].w);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / W) + eps);
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const float4 g = __ldg(g4 + i * 32 + lane);
        const float4 b = __ldg(b4 + i * 32 + lane);
        x[i].x = fmaf(x[i].x * rstd, g.x, b.x);
        x[i].y = fmaf(x[i].y * rstd, g.y, b.y);
        x[i].z = fmaf(x[i].z * rstd, g.z, b.z);
        x[i].w = fmaf(x[i].w * rstd, g.w, b.w);
    }
    return make_float2(mean, rstd);
}

// y = hi + lo of one row -> 4 W / 128 fp32 values per lane (same column mapping as a float4 row)
template <int W = H>
__device__ __forceinline__ void load_split_row(const __half* __restrict__ yhi, const __half* __restrict__ ylo, size_t row, int lane,
                                               float4 (&x)[Row<W>::V4]) {
    constexpr int V4 = Row<W>::V4;
    const uint2* h2 = reinterpret_cast<const uint2*>(yhi + row * W);
    const uint2* l2 = reinterpret_cast<const uint2*>(ylo + row * W);
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const uint2 hv = h2[i * 32 + lane], lv = l2[i * 32 + lane];
        const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&hv.x)), h1 = __half22float2(*reinterpret_cast<const __half2*>(&hv.y));
        const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&lv.x)), l1 = __half22float2(*reinterpret_cast<const __half2*>(&lv.y));
        x[i] = make_float4(h0.x + l0.x, h0.y + l0.y, h1.x + l1.x, h1.y + l1.y);
    }
}

// SEGS: `type` holds two rows and token p of item i takes row 1 when p >= segs[i] (the second segment of a
// [CLS] a [SEP] b [SEP] pair), row 0 otherwise; segs[i] is clamped to [0, S] (a device-resident caller's segs are not
// validated).  Without SEGS every token takes row 0 and `segs` is not read.
template <int W, bool SEGS>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ word, const float* __restrict__ pos,
             const float* __restrict__ type0, __half* __restrict__ yhi, __half* __restrict__ ylo, float2* __restrict__ stats,
             int n_tokens, int S, int vocab, const int32_t* __restrict__ segs) {
    constexpr int V4 = Row<W>::V4;
    const int lane = threadIdx.x & 31;
    const int tok = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
    if (tok >= n_tokens) return;
    int id = ids[tok];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);  // submit() rejects out-of-range ids; never read OOB
    const int p = tok % S;
    const float4* w4 = reinterpret_cast<const float4*>(word + static_cast<size_t>(id) * W);
    const float4* p4 = reinterpret_cast<const float4*>(pos + static_cast<size_t>(p) * W);
    const float* type_row = type0;
    if constexpr (SEGS) {
        int sg = segs[tok / S];
        sg = sg < 0 ? 0 : (sg > S ? S : sg);
        if (p >= sg) type_row += W;
    }
    const float4* t4 = reinterpret_cast<const float4*>(type_row);
    uint2* oh = reinterpret_cast<uint2*>(yhi + static_cast<size_t>(tok) * W);
    uint2* ol = reinterpret_cast<uint2*>(ylo + static_cast<size_t>(tok) * W);
    float ps = 0.f, pq = 0.f;  // lane i < V4 keeps partial i
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const float4 a = __ldg(w4 + i * 32 + lane);
        const float4 b = __ldg(p4 + i * 32 + lane);
        const float4 c = __ldg(t4 + i * 32 + lane);
        // HF order: (word + token_type) + position
        const float4 x = make_float4((a.x + c.x) + b.x, (a.y + c.y) + b.y, (a.z + c.z) + b.z, (a.w + c.w) + b.w);
        // the residual stream is kept PRE-LayerNorm as hi + lo; consumers fold / re-apply the LayerNorm
        const __half2 h0 = __floats2half2_rn(x.x, x.y), h1 = __floats2half2_rn(x.z, x.w);
        const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        oh[i * 32 + lane] = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
        ol[i * 32 + lane] = make_uint2(pack_half2(x.x - f0.x, x.y - f0.y), pack_half2(x.z - f1.x, x.w - f1.y));
        // (sum, M2 about its own mean) of this 128-column slice: float4 i of the 32 lanes is exactly slice i
        const float s = warp_sum((x.x + x.y) + (x.z + x.w));
        const float m = s * (1.0f / 128.0f);
        const float dx = x.x - m, dy = x.y - m, dz = x.z - m, dw = x.w - m;
        const float q = warp_sum((dx * dx + dy * dy) + (dz * dz + dw * dw));
        if (lane == i) { ps = s; pq = q; }
    }
    if (lane < V4) stats[static_cast<size_t>(tok) * V4 + lane] = make_float2(ps, pq);
}

template <int W>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
pool_normalize_kernel(const __half* __restrict__ yhi, const __half* __restrict__ ylo, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float* __restrict__ out, int n_items, int S, float eps) {
    constexpr int V4 = Row<W>::V4;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
    if (item >= n_items) return;
    float4 x[V4];
    load_split_row<W>(yhi, ylo, static_cast<size_t>(item) * S, lane, x);  // CLS row
    ln_inplace<W>(x, gamma, beta, eps, lane);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) q += (x[i].x * x[i].x + x[i].y * x[i].y) + (x[i].z * x[i].z + x[i].w * x[i].w);
    const float inv = 1.0f / fmaxf(sqrtf(warp_sum(q)), 1e-12f);  // torch.nn.functional.normalize eps
    float4* o4 = reinterpret_cast<float4*>(out + static_cast<size_t>(item) * W);  // may be peer memory
#pragma unroll
    for (int i = 0; i < V4; ++i)
        o4[i * 32 + lane] = make_float4(x[i].x * inv, x[i].y * inv, x[i].z * inv, x[i].w * inv);
}

// sentence-transformers' Pooling(mean) + Normalize: out[i] = L2normalise((1 / len_i) sum_{r < len_i} LN(hi + lo of row i S + r)),
// [CLS] and [SEP] included.  One block per item: warp w LayerNorms rows w, w + 8, w + 16, ... (the same load_split_row /
// ln_inplace as the CLS pool) and sums them in fp32 registers; the 8 warp sums are then added in warp order through shared
// memory.  The summation order is a function of len_i alone -- not of B, S, the grid or the replica -- so an item's embedding
// is bit-identical in any batch.  Rows len_i <= r < S are padding and are never read; len_i is clamped to [1, S] (lens may be
// a caller's unvalidated device array) and lens == NULL means every item is S long.
template <int W>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
mean_pool_normalize_kernel(const __half* __restrict__ yhi, const __half* __restrict__ ylo, const float* __restrict__ gamma,
                           const float* __restrict__ beta, const int32_t* __restrict__ lens, float* __restrict__ out, int S, float eps) {
    constexpr int V4 = Row<W>::V4;
    __shared__ __align__(16) float s_sum[WARPS_PER_BLOCK][W];
    __shared__ float s_red[WARPS_PER_BLOCK];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int item = blockIdx.x;
    int L = lens ? lens[item] : S;
    L = L < 1 ? 1 : (L > S ? S : L);
    float4 acc[V4];
#pragma unroll
    for (int i = 0; i < V4; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    auto add = [&](float4 (&x)[V4]) {
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            acc[i].x += x[i].x; acc[i].y += x[i].y; acc[i].z += x[i].z; acc[i].w += x[i].w;
        }
    };
    const size_t row0 = static_cast<size_t>(item) * S;
    int r = warp;
    // two rows in flight per warp (one block per item leaves few warps per SM to hide HBM latency); still added in row order
    for (; r + WARPS_PER_BLOCK < L; r += 2 * WARPS_PER_BLOCK) {
        float4 x[V4], x2[V4];
        load_split_row<W>(yhi, ylo, row0 + r, lane, x);
        load_split_row<W>(yhi, ylo, row0 + r + WARPS_PER_BLOCK, lane, x2);
        ln_inplace<W>(x, gamma, beta, eps, lane);
        add(x);
        ln_inplace<W>(x2, gamma, beta, eps, lane);
        add(x2);
    }
    if (r < L) {
        float4 x[V4];
        load_split_row<W>(yhi, ylo, row0 + r, lane, x);
        ln_inplace<W>(x, gamma, beta, eps, lane);
        add(x);
    }
#pragma unroll
    for (int i = 0; i < V4; ++i) *reinterpret_cast<float4*>(&s_sum[warp][i * 128 + 4 * lane]) = acc[i];
    __syncthreads();
    // column c = threadIdx.x + k * 256: the warp sums in warp order, then / len_i (sum / count, as Pooling(mean) divides)
    constexpr int PER_THREAD = (W + WARPS_PER_BLOCK * 32 - 1) / (WARPS_PER_BLOCK * 32);
    float v[PER_THREAD];
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < PER_THREAD; ++k) {
        const int c = threadIdx.x + k * WARPS_PER_BLOCK * 32;
        v[k] = 0.f;
        if (c < W) {
            float s = s_sum[0][c];
#pragma unroll
            for (int w = 1; w < WARPS_PER_BLOCK; ++w) s += s_sum[w][c];
            v[k] = s / static_cast<float>(L);
            q = fmaf(v[k], v[k], q);
        }
    }
    q = warp_sum(q);
    if (lane == 0) s_red[warp] = q;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS_PER_BLOCK; ++w) tot += s_red[w];
    const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);  // torch.nn.functional.normalize eps
    float* o = out + static_cast<size_t>(item) * W;  // may be peer memory
#pragma unroll
    for (int k = 0; k < PER_THREAD; ++k) {
        const int c = threadIdx.x + k * WARPS_PER_BLOCK * 32;
        if (c < W) o[c] = v[k] * inv;
    }
}

// BertForSequenceClassification's head (HF modeling_bert.py BertPooler + the classifier Linear): out[i] = W_c tanh(W_p x + b_p)
// + b_c, x = the last LayerNorm of the CLS row of item i, L raw logits per item (no sigmoid / softmax: the caller applies
// them).  Blocks walk items i = blockIdx.x, + gridDim.x, ...  Every warp LayerNorms its own copy of the CLS row (the
// load_split_row / ln_inplace of pool_normalize) and takes pooler rows n = warp, warp + 8, ...: a per-lane fma chain over the
// lane's columns then a warp_sum, so each h[n] is reduced in one fixed order.  The classifier rows j = warp, warp + 8, ... < L
// read h from shared memory in the same column layout.  Nothing depends on the grid, the batch or the replica, so an item's
// logits are bit-identical wherever it runs.  W_p fp32 [W, W] and W_c fp32 [L, W] are read by every item and stay L2-resident.
constexpr int CLS_HEAD_MAX_L = 64;
template <int W>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
cls_head_kernel(const __half* __restrict__ yhi, const __half* __restrict__ ylo, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ pool_w, const float* __restrict__ pool_b,
                const float* __restrict__ cls_w, const float* __restrict__ cls_b, float* __restrict__ out, int n_items, int S, int L,
                float eps) {
    constexpr int V4 = Row<W>::V4;
    __shared__ __align__(16) float s_h[W];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        float4 x[V4];
        load_split_row<W>(yhi, ylo, static_cast<size_t>(item) * S, lane, x);  // CLS row
        ln_inplace<W>(x, gamma, beta, eps, lane);
        for (int n = warp; n < W; n += WARPS_PER_BLOCK) {
            const float4* w4 = reinterpret_cast<const float4*>(pool_w + static_cast<size_t>(n) * W);
            float acc = 0.f;
#pragma unroll
            for (int i = 0; i < V4; ++i) {
                const float4 w = __ldg(w4 + i * 32 + lane);
                acc = fmaf(x[i].x, w.x, fmaf(x[i].y, w.y, fmaf(x[i].z, w.z, fmaf(x[i].w, w.w, acc))));
            }
            acc = warp_sum(acc);
            if (lane == 0) s_h[n] = tanhf(acc + __ldg(pool_b + n));
        }
        __syncthreads();
        float4 h[V4];
#pragma unroll
        for (int i = 0; i < V4; ++i) h[i] = *reinterpret_cast<const float4*>(&s_h[i * 128 + 4 * lane]);
        for (int j = warp; j < L; j += WARPS_PER_BLOCK) {
            const float4* w4 = reinterpret_cast<const float4*>(cls_w + static_cast<size_t>(j) * W);
            float acc = 0.f;
#pragma unroll
            for (int i = 0; i < V4; ++i) {
                const float4 w = __ldg(w4 + i * 32 + lane);
                acc = fmaf(h[i].x, w.x, fmaf(h[i].y, w.y, fmaf(h[i].z, w.z, fmaf(h[i].w, w.w, acc))));
            }
            acc = warp_sum(acc);
            if (lane == 0) out[static_cast<size_t>(item) * L + j] = acc + __ldg(cls_b + j);  // may be peer memory
        }
        __syncthreads();  // s_h is rewritten by the next item
    }
}

// ----------------------------------------------------------------------------------------------- ViT image tower (CLIP)
// Restates CLIPVisionEmbeddings.forward / the pooled head of CLIPVisionTransformer + visual_projection (HF modeling_clip.py)
// for the reference's image-embedding example (06_gpu_and_ml/embeddings/image_embeddings_infinity.py:76-77, 298-306).

// pixels fp32 [B, 3, img, img] -> A fp16 [B * T, 3 p p], T = (img/p)^2 + 1: row b*T is zero (the class token takes no patch),
// row b*T + 1 + (py*grid + px) holds patch (py, px) flattened (channel, row, column) -- the stride-p convolution as a GEMM.
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
im2col_kernel(const float* __restrict__ pixels, __half* __restrict__ a, int n_rows, int img, int p, int grid) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int T = grid * grid + 1, pd = 3 * p * p;
    const int b = row / T, tk = row % T;
    __half2* o = reinterpret_cast<__half2*>(a + static_cast<size_t>(row) * pd);
    if (tk == 0) {
        for (int e = lane; e < pd / 2; e += 32) o[e] = __floats2half2_rn(0.f, 0.f);
        return;
    }
    const int py = (tk - 1) / grid, px = (tk - 1) % grid;
    const float* base = pixels + static_cast<size_t>(b) * 3 * img * img + static_cast<size_t>(py * p) * img + px * p;
    for (int e = lane * 2; e < pd; e += 64) {
        const int c = e / (p * p), ky = (e / p) % p, kx = e % p;  // kx even: the pair stays inside one patch row
        const float2 v = *reinterpret_cast<const float2*>(base + (static_cast<size_t>(c) * img + ky) * img + kx);
        o[e / 2] = __floats2half2_rn(v.x, v.y);
    }
}

// row b*T + tk: e = (tk == 0 ? class_embedding : patch GEMM output) + position[tk]; h = pre_layrnorm(e) becomes the residual
// stream (hi + lo) together with its (sum, M2) partials -- the statistics LayerNorm1 of the first layer folds.
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
vit_embed_kernel(const __half* __restrict__ patch_out, const float* __restrict__ cls, const float* __restrict__ pos,
                 const float* __restrict__ gamma, const float* __restrict__ beta, __half* __restrict__ yhi, __half* __restrict__ ylo,
                 float2* __restrict__ stats, int n_rows, int T, float eps) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int tk = row % T;
    const uint2* p2 = reinterpret_cast<const uint2*>(patch_out + static_cast<size_t>(row) * H);
    const float4* c4 = reinterpret_cast<const float4*>(cls);
    const float4* q4 = reinterpret_cast<const float4*>(pos + static_cast<size_t>(tk) * H);
    float4 x[V4];
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        float4 v;
        if (tk == 0) {
            v = __ldg(c4 + i * 32 + lane);
        } else {
            const uint2 hv = p2[i * 32 + lane];
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hv.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&hv.y));
            v = make_float4(a.x, a.y, b.x, b.y);
        }
        const float4 q = __ldg(q4 + i * 32 + lane);
        x[i] = make_float4(v.x + q.x, v.y + q.y, v.z + q.z, v.w + q.w);
    }
    ln_inplace(x, gamma, beta, eps, lane);
    uint2* oh = reinterpret_cast<uint2*>(yhi + static_cast<size_t>(row) * H);
    uint2* ol = reinterpret_cast<uint2*>(ylo + static_cast<size_t>(row) * H);
    float ps = 0.f, pq = 0.f;
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const float4 v = x[i];
        const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
        const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        oh[i * 32 + lane] = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
        ol[i * 32 + lane] = make_uint2(pack_half2(v.x - f0.x, v.y - f0.y), pack_half2(v.z - f1.x, v.w - f1.y));
        const float sm = warp_sum((v.x + v.y) + (v.z + v.w));
        const float m = sm * (1.0f / 128.0f);
        const float dx = v.x - m, dy = v.y - m, dz = v.z - m, dw = v.w - m;
        const float q = warp_sum((dx * dx + dy * dy) + (dz * dz + dw * dw));
        if (lane == i) { ps = sm; pq = q; }
    }
    if (lane < V4) stats[static_cast<size_t>(row) * V4 + lane] = make_float2(ps, pq);
}

// One block per image: post_layernorm of the class-token row, visual projection [P, H], L2 normalise; row i is stored at
// out + i * P, possibly peer memory (the fused gather).
constexpr int VIT_POOL_MAX_P = 1024;
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
vit_pool_kernel(const __half* __restrict__ yhi, const __half* __restrict__ ylo, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ proj, float* __restrict__ out, int T, int P, float eps) {
    __shared__ float s_out[VIT_POOL_MAX_P];
    __shared__ float s_red[WARPS_PER_BLOCK];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int item = blockIdx.x;
    float4 x[V4];
    load_split_row(yhi, ylo, static_cast<size_t>(item) * T, lane, x);  // class-token row (every warp keeps its own copy)
    ln_inplace(x, gamma, beta, eps, lane);
    float sq = 0.f;
    for (int n = warp; n < P; n += WARPS_PER_BLOCK) {
        const float4* w4 = reinterpret_cast<const float4*>(proj + static_cast<size_t>(n) * H);
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            const float4 w = __ldg(w4 + i * 32 + lane);
            acc = fmaf(x[i].x, w.x, fmaf(x[i].y, w.y, fmaf(x[i].z, w.z, fmaf(x[i].w, w.w, acc))));
        }
        acc = warp_sum(acc);
        if (lane == 0) s_out[n] = acc;
        sq = fmaf(acc, acc, sq);  // identical on every lane after warp_sum
    }
    if (lane == 0) s_red[warp] = sq;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS_PER_BLOCK; ++w) tot += s_red[w];
    const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);
    float* o = out + static_cast<size_t>(item) * P;
    for (int n = threadIdx.x; n < P; n += WARPS_PER_BLOCK * 32) o[n] = s_out[n] * inv;
}

// ------------------------------------------------------------------------------------------ CLIP text tower (W = 512)
// Restates the pooled head of CLIPTextTransformer.forward + CLIPTextModelWithProjection.text_projection (HF modeling_clip.py)
// for infinity's `embed(sentences=...)` on the reference's CLIP model (image_embeddings_infinity.py:76-77, 298-306).
// One block per item.  The pooled position (see kernels.h) is reduced over the item's valid ids as (key, position) with the
// smallest position winning ties, so it does not depend on how the ids are strided over the threads.  Every warp then
// LayerNorms its own copy of the row and takes projection rows n = warp, warp + 8, ..., as vit_pool does.
constexpr int CLIP_TEXT_POOL_MAX_P = 1024;
template <int W>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
clip_text_pool_kernel(const __half* __restrict__ yhi, const __half* __restrict__ ylo, const int32_t* __restrict__ ids,
                      const int32_t* __restrict__ lens, const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* __restrict__ proj, float* __restrict__ out, int S, int P, float eps, int eos_id) {
    constexpr int V4 = Row<W>::V4;
    __shared__ float s_out[CLIP_TEXT_POOL_MAX_P];
    __shared__ float s_red[WARPS_PER_BLOCK];
    __shared__ int s_key[WARPS_PER_BLOCK], s_pos[WARPS_PER_BLOCK];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int item = blockIdx.x;
    int L = lens[item];
    L = L < 1 ? 1 : (L > S ? S : L);
    const int32_t* row_ids = ids + static_cast<size_t>(item) * S;
    // key of position p: its id (argmax branch) or 1 where id == eos_id (first-match branch); best = largest key, then the
    // smallest position.  First-match with no eos in the item: every key is 0 and position 0 wins.  A thread without positions
    // starts at (INT_MIN, 0), which no valid position loses to except at position 0 itself, so the winner is always in [0, L)
    // whatever the ids (a device-resident caller's ids are not validated).
    const bool argmax = eos_id == 2;
    int key = INT_MIN, pos = 0;
    for (int p = threadIdx.x; p < L; p += WARPS_PER_BLOCK * 32) {
        const int id = row_ids[p];
        const int k = argmax ? id : (id == eos_id ? 1 : 0);
        if (k > key) { key = k; pos = p; }  // p increases: a tie keeps the earlier position
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const int k2 = __shfl_xor_sync(0xffffffff, key, o), p2 = __shfl_xor_sync(0xffffffff, pos, o);
        if (k2 > key || (k2 == key && p2 < pos)) { key = k2; pos = p2; }
    }
    if (lane == 0) { s_key[warp] = key; s_pos[warp] = pos; }
    __syncthreads();
    key = s_key[0];
    pos = s_pos[0];
#pragma unroll
    for (int w = 1; w < WARPS_PER_BLOCK; ++w)
        if (s_key[w] > key || (s_key[w] == key && s_pos[w] < pos)) { key = s_key[w]; pos = s_pos[w]; }
    float4 x[V4];
    load_split_row<W>(yhi, ylo, static_cast<size_t>(item) * S + pos, lane, x);
    ln_inplace<W>(x, gamma, beta, eps, lane);  // final_layer_norm
    float sq = 0.f;
    for (int n = warp; n < P; n += WARPS_PER_BLOCK) {
        const float4* w4 = reinterpret_cast<const float4*>(proj + static_cast<size_t>(n) * W);
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < V4; ++i) {
            const float4 w = __ldg(w4 + i * 32 + lane);
            acc = fmaf(x[i].x, w.x, fmaf(x[i].y, w.y, fmaf(x[i].z, w.z, fmaf(x[i].w, w.w, acc))));
        }
        acc = warp_sum(acc);
        if (lane == 0) s_out[n] = acc;
        sq = fmaf(acc, acc, sq);  // identical on every lane after warp_sum
    }
    if (lane == 0) s_red[warp] = sq;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS_PER_BLOCK; ++w) tot += s_red[w];
    const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);
    float* o = out + static_cast<size_t>(item) * P;  // may be peer memory
    for (int n = threadIdx.x; n < P; n += WARPS_PER_BLOCK * 32) o[n] = s_out[n] * inv;
}

// Load-time weight preparation, one warp per output row n of W[N,K] (see kernels.h, "LNfold"):
//   gamma given: w_out[n,k] = fp16(w[n,k] gamma[k] - m_n),  m_n = mean_k(w[n,k] gamma[k])   (rows centred: the LayerNorm's mean
//                subtraction then happens inside the GEMM),  cvec[n] = sum_k w[n,k] beta[k] + bias[n]
//   gamma NULL : w_out[n,k] = fp16(w[n,k])
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
fold_ln_kernel(const float* __restrict__ w, const float* __restrict__ gamma, const float* __restrict__ beta,
               const float* __restrict__ bias, __half* __restrict__ w_out, float* __restrict__ cvec, int N, int K) {
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
    if (n >= N) return;
    const float* wr = w + static_cast<size_t>(n) * K;
    __half* orow = w_out + static_cast<size_t>(n) * K;
    float m = 0.f;
    if (gamma != nullptr) {
        float s = 0.f, c = 0.f;
        for (int k = lane * 2; k < K; k += 64) {
            const float2 wv = *reinterpret_cast<const float2*>(wr + k);
            s += fmaf(wv.x, __ldg(gamma + k), wv.y * __ldg(gamma + k + 1));
            c = fmaf(wv.x, __ldg(beta + k), fmaf(wv.y, __ldg(beta + k + 1), c));
        }
        m = warp_sum(s) / static_cast<float>(K);
        c = warp_sum(c);
        if (lane == 0 && cvec != nullptr) cvec[n] = c + (bias != nullptr ? bias[n] : 0.f);
    }
    for (int k = lane * 2; k < K; k += 64) {
        const float2 wv = *reinterpret_cast<const float2*>(wr + k);
        const float g0 = gamma != nullptr ? __ldg(gamma + k) : 1.f, g1 = gamma != nullptr ? __ldg(gamma + k + 1) : 1.f;
        *reinterpret_cast<__half2*>(orow + k) = __floats2half2_rn(fmaf(wv.x, g0, -m), fmaf(wv.y, g1, -m));
    }
}

// SPLADE head, one warp per row of u (fp16, W wide): the (sum, M2 about its own mean) partial of each 128-column slice, from
// the fp16 values the decoder GEMM reads, as embed_kernel computes them; and every thread zeroes its grid-stride share of
// the decoder's max buffer vmax [n_max].
template <int W>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32)
mlm_ln_stats_kernel(const __half* __restrict__ u, float2* __restrict__ stats, uint32_t* __restrict__ vmax, int n_rows, size_t n_max) {
    constexpr int V4 = Row<W>::V4;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x, nth = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = tid; i < n_max / 4; i += nth) reinterpret_cast<uint4*>(vmax)[i] = make_uint4(0, 0, 0, 0);
    for (size_t i = n_max / 4 * 4 + tid; i < n_max; i += nth) vmax[i] = 0;
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const uint2* u2 = reinterpret_cast<const uint2*>(u + static_cast<size_t>(row) * W);
    float ps = 0.f, pq = 0.f;  // lane i < V4 keeps partial i
#pragma unroll
    for (int i = 0; i < V4; ++i) {
        const uint2 hv = u2[i * 32 + lane];
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hv.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&hv.y));
        const float s = warp_sum((a.x + a.y) + (b.x + b.y));
        const float m = s * (1.0f / 128.0f);
        const float dx = a.x - m, dy = a.y - m, dz = b.x - m, dw = b.y - m;
        const float q = warp_sum((dx * dx + dy * dy) + (dz * dz + dw * dw));
        if (lane == i) { ps = s; pq = q; }
    }
    if (lane < V4) stats[static_cast<size_t>(row) * V4 + lane] = make_float2(ps, pq);
}

// blockIdx.y = item: out[item * vocab + v] = log1p(max) for v < vocab; log1pf (not __logf(1 + x)): the small values decide
// which words are non-zero.
__global__ void __launch_bounds__(256)
splade_finalize_kernel(const uint32_t* __restrict__ vmax, float* __restrict__ out, int vpad, int vocab) {
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v >= vocab) return;
    const size_t item = blockIdx.y;
    out[item * vocab + v] = log1pf(__uint_as_float(vmax[item * vpad + v]));
}

// blockIdx.y = shard.  Copies ids[item_begin*S .. (item_begin+item_count)*S) and the matching lens (and, SEGS, segment
// starts) to the shard's input slot; dst pointers of remote shards are peer-mapped, so the stores cross NVLink directly.
template <bool SEGS>
__global__ void __launch_bounds__(256)
scatter_kernel(const int32_t* __restrict__ src_ids, const int32_t* __restrict__ src_lens, const ScatterPlan plan,
               const int32_t* __restrict__ src_segs) {
    const int sh = blockIdx.y;
    const int cnt = plan.item_count[sh];
    if (cnt <= 0) return;
    const int S = plan.S;
    const size_t n = static_cast<size_t>(cnt) * S;
    const int32_t* s = src_ids + static_cast<size_t>(plan.item_begin[sh]) * S;
    int32_t* d = plan.dst_ids[sh];
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    if ((((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15) == 0)) {
        const size_t n4 = n / 4;
        for (size_t i = tid; i < n4; i += stride) reinterpret_cast<int4*>(d)[i] = reinterpret_cast<const int4*>(s)[i];
        for (size_t i = n4 * 4 + tid; i < n; i += stride) d[i] = s[i];
    } else {
        for (size_t i = tid; i < n; i += stride) d[i] = s[i];
    }
    for (size_t i = tid; i < static_cast<size_t>(cnt); i += stride) plan.dst_lens[sh][i] = src_lens[plan.item_begin[sh] + i];
    if constexpr (SEGS)
        for (size_t i = tid; i < static_cast<size_t>(cnt); i += stride) plan.dst_segs[sh][i] = src_segs[plan.item_begin[sh] + i];
}

}  // namespace rw

cudaError_t launch_embed(const int32_t* ids, const float* word, const float* pos, const float* type0, __half* yhi, __half* ylo,
                         float2* stats, int n_tokens, int S, int vocab, int width, cudaStream_t stream, const int32_t* segs) {
    const int grid = (n_tokens + rw::WARPS_PER_BLOCK - 1) / rw::WARPS_PER_BLOCK;
    const int block = rw::WARPS_PER_BLOCK * 32;
    if (segs) {  // token pairs: BERT classifiers only (768, 384, 1024)
        if (width == 768) rw::embed_kernel<768, true><<<grid, block, 0, stream>>>(ids, word, pos, type0, yhi, ylo, stats, n_tokens, S, vocab, segs);
        else if (width == 384) rw::embed_kernel<384, true><<<grid, block, 0, stream>>>(ids, word, pos, type0, yhi, ylo, stats, n_tokens, S, vocab, segs);
        else if (width == 1024) rw::embed_kernel<1024, true><<<grid, block, 0, stream>>>(ids, word, pos, type0, yhi, ylo, stats, n_tokens, S, vocab, segs);
        else return cudaErrorInvalidValue;
        return cudaGetLastError();
    }
    if (width == 768) rw::embed_kernel<768, false><<<grid, block, 0, stream>>>(ids, word, pos, type0, yhi, ylo, stats, n_tokens, S, vocab, nullptr);
    else if (width == 384) rw::embed_kernel<384, false><<<grid, block, 0, stream>>>(ids, word, pos, type0, yhi, ylo, stats, n_tokens, S, vocab, nullptr);
    else if (width == 1024) rw::embed_kernel<1024, false><<<grid, block, 0, stream>>>(ids, word, pos, type0, yhi, ylo, stats, n_tokens, S, vocab, nullptr);
    else if (width == 512) rw::embed_kernel<512, false><<<grid, block, 0, stream>>>(ids, word, pos, type0, yhi, ylo, stats, n_tokens, S, vocab, nullptr);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

cudaError_t launch_cls_head(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, const float* pool_w,
                            const float* pool_b, const float* cls_w, const float* cls_b, float* out, int n_items, int S, int L, float eps,
                            int width, cudaStream_t stream, int ctas) {
    if (n_items < 1 || S < 1 || L < 1 || L > rw::CLS_HEAD_MAX_L || ctas < 0) return cudaErrorInvalidValue;
    const int grid = ctas == 0 || ctas > n_items ? n_items : ctas;
    const int block = rw::WARPS_PER_BLOCK * 32;
    if (width == 768) rw::cls_head_kernel<768><<<grid, block, 0, stream>>>(yhi, ylo, gamma, beta, pool_w, pool_b, cls_w, cls_b, out, n_items, S, L, eps);
    else if (width == 384) rw::cls_head_kernel<384><<<grid, block, 0, stream>>>(yhi, ylo, gamma, beta, pool_w, pool_b, cls_w, cls_b, out, n_items, S, L, eps);
    else if (width == 1024) rw::cls_head_kernel<1024><<<grid, block, 0, stream>>>(yhi, ylo, gamma, beta, pool_w, pool_b, cls_w, cls_b, out, n_items, S, L, eps);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

cudaError_t launch_pool_normalize(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, float* out,
                                  int n_items, int S, float eps, int width, cudaStream_t stream) {
    const int grid = (n_items + rw::WARPS_PER_BLOCK - 1) / rw::WARPS_PER_BLOCK;
    if (width == 768) rw::pool_normalize_kernel<768><<<grid, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(yhi, ylo, gamma, beta, out, n_items, S, eps);
    else if (width == 384) rw::pool_normalize_kernel<384><<<grid, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(yhi, ylo, gamma, beta, out, n_items, S, eps);
    else if (width == 1024) rw::pool_normalize_kernel<1024><<<grid, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(yhi, ylo, gamma, beta, out, n_items, S, eps);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

cudaError_t launch_mean_pool_normalize(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, const int32_t* lens,
                                       float* out, int n_items, int S, float eps, int width, cudaStream_t stream) {
    if (n_items < 1 || S < 1) return cudaErrorInvalidValue;
    const int block = rw::WARPS_PER_BLOCK * 32;
    if (width == 768) rw::mean_pool_normalize_kernel<768><<<n_items, block, 0, stream>>>(yhi, ylo, gamma, beta, lens, out, S, eps);
    else if (width == 384) rw::mean_pool_normalize_kernel<384><<<n_items, block, 0, stream>>>(yhi, ylo, gamma, beta, lens, out, S, eps);
    else if (width == 1024) rw::mean_pool_normalize_kernel<1024><<<n_items, block, 0, stream>>>(yhi, ylo, gamma, beta, lens, out, S, eps);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

cudaError_t launch_im2col(const float* pixels, __half* a, int n_items, int img, int p, cudaStream_t stream) {
    const int grid_sz = img / p, T = grid_sz * grid_sz + 1;
    if (img % p != 0 || (3 * p * p) % 64 != 0 || p % 2 != 0) return cudaErrorInvalidValue;
    const int rows = n_items * T;
    rw::im2col_kernel<<<(rows + rw::WARPS_PER_BLOCK - 1) / rw::WARPS_PER_BLOCK, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(pixels, a, rows, img, p, grid_sz);
    return cudaGetLastError();
}

cudaError_t launch_vit_embed(const __half* patch_out, const float* cls, const float* pos, const float* gamma, const float* beta,
                             __half* yhi, __half* ylo, float2* stats, int n_rows, int T, float eps, cudaStream_t stream) {
    rw::vit_embed_kernel<<<(n_rows + rw::WARPS_PER_BLOCK - 1) / rw::WARPS_PER_BLOCK, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(
        patch_out, cls, pos, gamma, beta, yhi, ylo, stats, n_rows, T, eps);
    return cudaGetLastError();
}

cudaError_t launch_vit_pool(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, const float* proj, float* out,
                            int n_items, int T, int P, float eps, cudaStream_t stream) {
    if (P < 1 || P > rw::VIT_POOL_MAX_P) return cudaErrorInvalidValue;
    rw::vit_pool_kernel<<<n_items, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(yhi, ylo, gamma, beta, proj, out, T, P, eps);
    return cudaGetLastError();
}

cudaError_t launch_clip_text_pool(const __half* yhi, const __half* ylo, const int32_t* ids, const int32_t* lens, const float* gamma,
                                  const float* beta, const float* proj, float* out, int n_items, int S, int P, float eps, int eos_id,
                                  cudaStream_t stream) {
    if (n_items < 1 || S < 1 || P < 1 || P > rw::CLIP_TEXT_POOL_MAX_P) return cudaErrorInvalidValue;
    rw::clip_text_pool_kernel<512><<<n_items, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(yhi, ylo, ids, lens, gamma, beta, proj, out, S, P, eps,
                                                                                     eos_id);
    return cudaGetLastError();
}

cudaError_t launch_fold_ln(const float* w, const float* gamma, const float* beta, const float* bias, __half* w_out, float* cvec,
                           int N, int K, cudaStream_t stream) {
    if (K % 64 != 0 || N < 1) return cudaErrorInvalidValue;
    const int grid = (N + rw::WARPS_PER_BLOCK - 1) / rw::WARPS_PER_BLOCK;
    rw::fold_ln_kernel<<<grid, rw::WARPS_PER_BLOCK * 32, 0, stream>>>(w, gamma, beta, bias, w_out, cvec, N, K);
    return cudaGetLastError();
}

cudaError_t launch_mlm_ln_stats(const __half* u, float2* stats, uint32_t* vmax, int n_rows, size_t n_max, int width, cudaStream_t stream) {
    if (n_rows < 1 || (n_max > 0 && vmax == nullptr)) return cudaErrorInvalidValue;
    const int grid = (n_rows + rw::WARPS_PER_BLOCK - 1) / rw::WARPS_PER_BLOCK;
    const int block = rw::WARPS_PER_BLOCK * 32;
    if (width == 768) rw::mlm_ln_stats_kernel<768><<<grid, block, 0, stream>>>(u, stats, vmax, n_rows, n_max);
    else if (width == 384) rw::mlm_ln_stats_kernel<384><<<grid, block, 0, stream>>>(u, stats, vmax, n_rows, n_max);
    else if (width == 1024) rw::mlm_ln_stats_kernel<1024><<<grid, block, 0, stream>>>(u, stats, vmax, n_rows, n_max);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

cudaError_t launch_splade_finalize(const uint32_t* vmax, float* out, int n_items, int vpad, int vocab, cudaStream_t stream) {
    if (n_items < 1 || n_items > 65535 || vocab < 1 || vocab > vpad) return cudaErrorInvalidValue;
    rw::splade_finalize_kernel<<<dim3((vocab + 255) / 256, n_items), 256, 0, stream>>>(vmax, out, vpad, vocab);
    return cudaGetLastError();
}

cudaError_t launch_scatter(const int32_t* src_ids, const int32_t* src_lens, const ScatterPlan& plan,
                           cudaStream_t stream, const int32_t* src_segs) {
    if (plan.n_shards < 1 || plan.n_shards > ScatterPlan::MAX_SHARDS) return cudaErrorInvalidValue;
    int max_cnt = 0;
    for (int i = 0; i < plan.n_shards; ++i) max_cnt = plan.item_count[i] > max_cnt ? plan.item_count[i] : max_cnt;
    if (max_cnt == 0) return cudaSuccess;
    const size_t n4 = (static_cast<size_t>(max_cnt) * plan.S + 3) / 4;
    int gx = static_cast<int>((n4 + 255) / 256);
    gx = gx < 1 ? 1 : (gx > 132 * 4 ? 132 * 4 : gx);
    if (src_segs) rw::scatter_kernel<true><<<dim3(gx, plan.n_shards), 256, 0, stream>>>(src_ids, src_lens, plan, src_segs);
    else rw::scatter_kernel<false><<<dim3(gx, plan.n_shards), 256, 0, stream>>>(src_ids, src_lens, plan, nullptr);
    return cudaGetLastError();
}

}  // namespace b200
