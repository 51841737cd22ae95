// Internal launch interface between the engine (host C++) and the sm_90a kernels.
// Every launch_* function refuses operands outside the contract its comment documents with cudaErrorInvalidValue, having
// enqueued nothing.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

enum GemmEpilogue : int {
    EPI_BIAS_F16 = 0,       // out fp16 = LNfold(acc) + bias                     (fused QKV projection)
    EPI_BIAS_GELU_F16 = 1,  // out fp16 = gelu_erf(LNfold(acc) + bias)           (FFN up-projection)
    EPI_BIAS_RES_SPLIT = 2, // y (fp16 hi + fp16 lo, in place) = acc + bias + LN(y)  (attention-out / FFN down) + row statistics
    EPI_BIAS_QGELU_F16 = 3, // out fp16 = quick_gelu(LNfold(acc) + bias), x * sigmoid(1.702 x)   (CLIP MLP up-projection)
    EPI_SPLADE_MAX = 4,     // per item and column: max over the item's valid rows of relu(LNfold(acc) + bias)   (SPLADE decoder)
    EPI_ROPE_F16 = 5,       // out fp16 = rotary(LNfold(acc) + bias) on the Q and K columns       (nomic-bert QKV projection)
    EPI_SWIGLU_F16 = 6,     // out fp16 [M, N/2] = silu(g) u of interleaved gate / up columns    (nomic-bert FFN up-projection)
};

// Four text geometries: bge-base (hidden 768, 12 heads of 64, inter 3072), bge-small (hidden 384, 12 heads of 32, inter 1536),
// bge-large (hidden 1024, 16 heads of 64, inter 4096) and the CLIP text tower (hidden 512, 8 heads of 64, inter 2048); the ViT
// tower is 768 wide.  The constants below are bge-base's:
// workspaces are sized by them for the runtime's row capacity.  bge-small uses the same buffers densely at its own widths;
// bge-large, 4/3 of bge-base in every width, uses them densely for 3/4 of the rows (the engine's per-model row capacity).
constexpr int HIDDEN = 768;
constexpr int HEADS = 12;  // bge-base, bge-small and the ViT tower
constexpr int QKV_DIM = 3 * HIDDEN;
constexpr int STAT_PARTS = HIDDEN / 128;  // row statistics travel as one (sum, M2) partial per 128 columns: 6 (768), 3 (384), 8 (1024) or 4 (512)

// One-time per-device setup (dynamic shared memory opt-in for every kernel). Call with the device current.
cudaError_t kernels_init_device();

// The residual stream lives in HBM as y = hi + lo (two fp16 arrays, 22 mantissa bits together), stored PRE-LayerNorm, with
// the row statistics of the LayerNorm that applies to it as width / 128 partials per row: (sum, M2 about the partial's own
// mean) over each 128-column slice, written by whoever produced the row (embedding kernel or a residual GEMM epilogue).
// No kernel ever materialises LN(y):
//   * a GEMM that consumes LN(y) reads `hi` as its fp16 A operand against W'' = fp16(gamma o W - rowmean(gamma o W)): gamma folded
//     into the weight's columns and every row centred at load time, so that sum_k (y_k - mean) W''_nk = sum_k y_k W''_nk and the
//     row mean never has to be subtracted; its epilogue applies  rstd * acc + (W beta + b)   -- "LNfold";
//   * a GEMM that adds the residual LN(y) re-applies (y - mean) * rstd * gamma + beta in its epilogue.
//
// C[M,N] = epi(A[M,K] . W[N,K]^T).  A and W move by TMA:
//   ta  : fp16 A   {K, rows>=M}  box {64,128} SW128     tb  : fp16 W {K, N} box {64,128} SW128
//   EPI 0/1/3: out = fp16 [M, N] row-major, written by TMA stores through oe (required): a map over out, {N, M} -- exactly M
//              rows, so that the stores clip the last tile's rows past M -- box {64, 64} SW128; e.stats_in (or NULL: plain
//              acc + bias), e.bias
//   EPI 2    : out = hi, out_lo = lo, both fp16 [M, N] row-major (read and written in place); res (required) holds TMA maps
//              over the same hi and lo, {N, rows>=M} box {64,128} SW128 like ta, through which the tile's residual is read;
//              e.stats_in + e.ln_gamma/e.ln_beta describe the LayerNorm of the residual (stats_in NULL: the residual is added
//              as is); e.stats_out receives the partials of the new rows (N / 128 per row; must not alias stats_in: other tiles
//              still read those).  EPI 0/1/3 take out_lo and res NULL, EPI 2 oe NULL.
//   N % 128 == 0, K % 64 == 0; rows past M are neither read from out nor written.  Tiles are 128 x 256 when N % 256 == 0,
//   else 128 x 128.  e.parts_in (with stats_in) must be the LayerNorm'd width / 128, that width being 768 or 384 (K for
//   EPI 0/1/3, N for EPI 2), 1024 for EPI 0/1/2 with N % 256 == 0, or 512 for EPI 0/3 with N % 256 == 0.  ta's map may end at M rows or run past them: a tile's A rows past M only feed rows no store
//   reaches.
//   The kernel runs as 2-CTA clusters (two m-tiles sharing one W tile):  min(tile pairs, sm_count / 2, the clusters that
//   fit at once) clusters, at least one -- sm_count bounds the CTAs from above, rounded down to whole clusters, except that
//   sm_count = 1 still launches one cluster of 2.  The result does not depend on sm_count.  ctas (optional) receives the
//   number of CTAs launched.
struct GemmEpi {
    const float* bias;        // [N]
    const float2* stats_in;   // [rows][parts_in]
    int parts_in;             // partials per row of stats_in (LayerNorm width / 128)
    const float* ln_gamma;    // [N] EPI 2
    const float* ln_beta;     // [N] EPI 2
    float2* stats_out;        // [rows][N / 128] EPI 2 (may be NULL)
    float eps;
};
// EPI 2's residual stream as the kernel reads it: hi and lo, each {N, rows} box {64, 128} SW128
struct ResEpi {
    CUtensorMap hi, lo;
};
// EPI 0/1/3's output as the kernel stores it: {N, M} box {64, 64} SW128
struct OutEpi {
    CUtensorMap out;
};
cudaError_t launch_gemm(int epi, const CUtensorMap& ta, const CUtensorMap& tb, __half* out, __half* out_lo, const ResEpi* res,
                        const OutEpi* oe, const GemmEpi& e, int M, int N, int K, int sm_count, cudaStream_t stream, int* ctas = nullptr);

// SPLADE's vocabulary max (EPI_SPLADE_MAX): the decoder GEMM C = LNfold(A . W^T) + bias over rows of items padded to S tokens
// (S % 64 == 0, M = B S), never stored.  Instead, for item i and column n < vocab,
//   vmax[i * N + n] = max(vmax[i * N + n], bits(max over rows r of item i with r % S < lens[i] of max(C[r, n], 0)))
// by red.global.max.u32 on the fp32 bits (exact and order-independent for values >= 0), one per 64-row consumer half and
// column, none for a zero.  vmax must hold zeros (or earlier maxima) for the B items; columns >= vocab are never written.
// e.stats_in is required (the LayerNorm of A, K wide: 768, 384 or 1024); N % 256 == 0, 1 <= vocab <= N, S >= 64 a multiple of 64
// dividing M.  lens[i] is clamped to [0, S].
struct SpladeEpi {
    const int32_t* lens;  // [B]
    int S;
    uint32_t* vmax;       // [B, N]
    int vocab;
};
cudaError_t launch_gemm_splade(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpi& e, const SpladeEpi& sp, int M, int N, int K,
                               int sm_count, cudaStream_t stream, int* ctas = nullptr);

// Rotary embedding of the QKV projection (EPI_ROPE_F16): out = fp16 [M, N] of v = LNfold(acc) + bias (e.stats_in NULL: acc +
// bias), and on columns n < rot_cols (Q | K; a multiple of 256) the pair (d, d + 32) of every 64-column head, v_d and
// v_{d+32}, becomes (v_d cos - v_{d+32} sin, v_{d+32} cos + v_d sin) with (cos, sin) = table[(row % S) * 32 + d] (HF's
// rotate_half, not interleaved).  table: fp32 [>= S rows][32] float2, one row per position.  K = 768 (6 partials), N % 256 == 0,
// S >= 64 a multiple of 64, rot_cols <= N.
struct RopeEpi {
    const float2* table;
    int S;         // padded length of the wave's items: row r is position r % S
    int rot_cols;  // 2 H
};
cudaError_t launch_gemm_rope(const CUtensorMap& ta, const CUtensorMap& tb, __half* out, const GemmEpi& e, const RopeEpi& rp, int M, int N,
                             int K, int sm_count, cudaStream_t stream, int* ctas = nullptr);

// SwiGLU up-projection (EPI_SWIGLU_F16): W [N, K] holds gate and up rows interleaved in groups of 8 (rows 16k .. 16k+7 = gate
// rows 8k .. 8k+7, rows 16k+8 .. 16k+15 = up rows 8k .. 8k+7); out = fp16 [M, N / 2], out[r, 8k + i] = silu(g) u with g, u the
// LNfold(acc) + bias of W rows 16k + i and 16k + 8 + i.  K = 768 (6 partials), N % 256 == 0.
cudaError_t launch_gemm_swiglu(const CUtensorMap& ta, const CUtensorMap& tb, __half* out, const GemmEpi& e, int M, int N, int K, int sm_count,
                               cudaStream_t stream, int* ctas = nullptr);

// gamma != NULL: w_out[n,k] = fp16(w[n,k] gamma[k] - mean_k(w[n,:] gamma)), cvec[n] = sum_k w[n,k] beta[k] + bias[n]
// gamma == NULL: w_out = fp16(w) (cvec untouched).  N >= 1, K % 64 == 0.
cudaError_t launch_fold_ln(const float* w, const float* gamma, const float* beta, const float* bias, __half* w_out, float* cvec,
                           int N, int K, cudaStream_t stream);

// Multi-head self-attention over a padded batch of `heads` heads of head_dim, H = heads head_dim: (head_dim, heads) is
// (64, 12), (32, 12) or (64, 16); causal (key k masked for query row q when k > q, CLIP's text tower): (64, 8) only.  1 <= S <= 512.  qkv fp16 [B, S, 3H] (Q | K | V, head-major within each), lens[B] valid keys per item, ctx
// fp16 [B*S, H].  tq: 3D map over qkv {3H, S, B}, tctx: 3D map over ctx {H, S, B}; both box {head_dim, 128, 1}, 128B (d = 64)
// or 64B (d = 32) swizzle.  Persistent: min(units, sm_count) CTAs walk the (item, head[, query tile]) units.
cudaError_t launch_attention(const CUtensorMap& tq, const CUtensorMap& tctx, const int32_t* lens, int B, int S, int sm_count,
                             cudaStream_t stream, int head_dim, int heads, bool causal);

// Streaming K/V attention (nomic-bert: 12 heads of 64, no mask but the length), any S with 64 <= S <= 8192 and S % 64 == 0.
// qkv and tq as for launch_attention (tq: 3D map over qkv {3H, S, B}, box {64, 128, 1}, 128B swizzle); ctx fp16 [B*S, 768]
// written directly (rows past S are not written).  Persistent: min(B 12 ceil(S / 128), sm_count) CTAs walk the (item, head,
// 128-row query tile) units; a unit reads only its item's ceil(len / 128) key tiles.  At S <= 512 the result is bit-identical
// to launch_attention's with (64, 12).
cudaError_t launch_attention_stream(const CUtensorMap& tq, __half* ctx, const int32_t* lens, int B, int S, int sm_count, cudaStream_t stream);

// Text row kernels on rows of `width` (768, 384 or 1024; embed also 512) columns.
// word + position + token_type embedding gather -> y = hi + lo (pre-LN residual stream) + the row's statistic partials.
// segs NULL: every token takes type row 0.  segs [n_tokens / S] (768, 384, 1024 only): token p of item i takes type row 1
// (type0 + width) when p >= segs[i], clamped to [0, S] on the device, else row 0 -- the second segment of a sentence pair.
cudaError_t launch_embed(const int32_t* ids, const float* word, const float* pos, const float* type0, __half* yhi, __half* ylo,
                         float2* stats, int n_tokens, int S, int vocab, int width, cudaStream_t stream, const int32_t* segs = nullptr);

// BertForSequenceClassification's head: out + i * L = W_c tanh(W_p LN(hi + lo of row i * S) + b_p) + b_c, L raw logits per
// item (1 <= L <= 64), pool_w fp32 [width, width], cls_w fp32 [L, width].  Reductions run in a fixed order per item, so the
// logits do not depend on the batch, the grid or the replica.  ctas: the most blocks launched (0 = one per item; blocks walk
// the items).  `out` may be peer memory.
cudaError_t launch_cls_head(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, const float* pool_w,
                            const float* pool_b, const float* cls_w, const float* cls_b, float* out, int n_items, int S, int L, float eps,
                            int width, cudaStream_t stream, int ctas = 0);

// SPLADE head, between the transform GEMM and the decoder GEMM: the (sum, M2) partial of every 128-column slice of the fp16 rows
// u [n_rows, width] (the values the decoder GEMM reads) into stats [n_rows][width / 128], and vmax [n_max] zeroed (the
// decoder's max buffer of the wave's items).  width 768, 384 or 1024.
cudaError_t launch_mlm_ln_stats(const __half* u, float2* stats, uint32_t* vmax, int n_rows, size_t n_max, int width, cudaStream_t stream);

// out[i * vocab + v] = log1pf(fp32 bits vmax[i * vpad + v]) for v < vocab: SPLADE's log(1 + relu) applied once per (item, word)
// after the max (both are monotone).  1 <= n_items <= 65535 (the grid's y), 1 <= vocab <= vpad.  `out` may be peer memory.
cudaError_t launch_splade_finalize(const uint32_t* vmax, float* out, int n_items, int vpad, int vocab, cudaStream_t stream);

// final LayerNorm of the CLS row of every item + L2 normalise; row i is stored at out + i * width,
// where `out` may be a peer-mapped pointer into the root GPU's gather buffer (the fused gather).
cudaError_t launch_pool_normalize(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, float* out,
                                  int n_items, int S, float eps, int width, cudaStream_t stream);

// mean pooling (sentence-transformers Pooling(mean)) + L2 normalise: out + i * width = normalise((1 / len_i) sum over rows
// i * S + r, r < len_i, of the final LayerNorm of hi + lo), len_i = lens[i] clamped to [1, S] (lens NULL: S).  Rows past
// len_i are never read.  One block per item; the summation order depends on len_i only.  `out` may be peer memory.
cudaError_t launch_mean_pool_normalize(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, const int32_t* lens,
                                       float* out, int n_items, int S, float eps, int width, cudaStream_t stream);

// ViT image tower (CLIP): pixels fp32 [n, 3, img, img] -> im2col A fp16 [n*T, 3 p p] (class-token rows zero); patch GEMM output +
// class / position embeddings + pre_layrnorm -> residual stream + statistics; pooled head: post_layernorm(class token) ->
// projection [P, 768] -> L2 normalise, stored at out + i * P (possibly peer memory), 1 <= P <= 1024.
cudaError_t launch_im2col(const float* pixels, __half* a, int n_items, int img, int p, cudaStream_t stream);
cudaError_t launch_vit_embed(const __half* patch_out, const float* cls, const float* pos, const float* gamma, const float* beta,
                             __half* yhi, __half* ylo, float2* stats, int n_rows, int T, float eps, cudaStream_t stream);
cudaError_t launch_vit_pool(const __half* yhi, const __half* ylo, const float* gamma, const float* beta, const float* proj, float* out,
                            int n_items, int T, int P, float eps, cudaStream_t stream);

// CLIP text tower's pooled head, one block per item: the pooled row p_i of item i is chosen from its ids[i * S .. + len_i)
// (len_i = lens[i] clamped to [1, S]; ids past it are never read): eos_id == 2 (HF's legacy branch, the original openai
// configs): the first position of the largest id; otherwise the first position equal to eos_id, 0 when there is none.  Then
// final_layer_norm(hi + lo of row i * S + p_i) -> projection [P, 512] -> L2 normalise, stored at out + i * P (possibly peer
// memory).  1 <= P <= 1024.
cudaError_t launch_clip_text_pool(const __half* yhi, const __half* ylo, const int32_t* ids, const int32_t* lens, const float* gamma,
                                  const float* beta, const float* proj, float* out, int n_items, int S, int P, float eps, int eos_id,
                                  cudaStream_t stream);

// Root-side scatter of a wave's token ids / lengths (and, src_segs given, segment starts into dst_segs) into each shard's
// (possibly peer) input slot.
struct ScatterPlan {
    static constexpr int MAX_SHARDS = 16;
    int n_shards;
    int S;  // padded length of every item in the wave
    int32_t* dst_ids[MAX_SHARDS];
    int32_t* dst_lens[MAX_SHARDS];
    int item_begin[MAX_SHARDS];
    int item_count[MAX_SHARDS];
    int32_t* dst_segs[MAX_SHARDS];  // read only when launch_scatter is given src_segs
};
cudaError_t launch_scatter(const int32_t* src_ids, const int32_t* src_lens, const ScatterPlan& plan,
                           cudaStream_t stream, const int32_t* src_segs = nullptr);

}  // namespace b200

#ifdef __CUDACC__
#include <utility>
// Launch with programmatic stream serialisation: the kernel's CTAs may be scheduled while the previous kernel of the
// stream drains (see ptx.cuh: griddep_launch_dependents / griddep_wait); the kernel itself waits before it reads anything
// the previous kernel wrote.  A kernel declared with __cluster_dims__ (the GEMM) is launched in clusters of that shape; the
// grid must then be a whole number of clusters.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
}
#endif
