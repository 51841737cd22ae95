/* b200rt debug / test entry points: single kernels behind host buffers so that tests/ can compare each
 * one against the oracle.  Not part of the drop-in boundary; same conventions as b200rt.h.           */
#ifndef B200RT_DEBUG_H
#define B200RT_DEBUG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* out[M,N] = epi(A[M,K] . W[N,K]^T + bias (+ resid)) on replica 0, N % 128 == 0, K % 64 == 0.  a, w: fp16 bit patterns (uint16),
 * bias fp32 [N], resid fp32 [M,N] or NULL.  epi: 0 bias->fp16 out, 1 bias+gelu->fp16 out, 2 bias+resid->fp32
 * out (the residual travels through the kernel as fp16 hi + fp16 lo; out = hi + lo), 3 bias+quick_gelu->fp16 out.
 * out is uint16 [M,N] for epi 0/1/3 and float [M,N] for epi 2.  ms_out (optional): device time of `iters` back-to-back
 * launches divided by iters.
 * LayerNorm in the epilogue (optional; all NULL = none): ln_stats = [M][parts] (sum, M2) float pairs, one per 128 columns
 * of the LayerNorm'd row (parts = K/128 for epi 0/1/3, N/128 for epi 2; that width must be 768 or 384, or 1024 for epi 0/1/2
 * with N % 256 == 0; see b200rt_debug_gemm_ex for 512).
 *   epi 0/1/3: `a` is the PRE-LayerNorm row in fp16, `w` = fp16(gamma o W with every row centred: sum_k w[n,k] = 0),
 *            bias = W beta + b:  out = epi(rstd * acc + bias)
 *   epi 2  : out = acc + bias + ((resid - mean) * rstd * ln_gamma + ln_beta) (ln_stats NULL: acc + bias + resid);
 *            stats_out (optional) receives [M][N/128] (sum, M2) partials of the new rows.
 * sms: the most CTAs the persistent kernel is launched with (0 = the device's SM count, else 1..SM count; anything else
 * is B200RT_E_INVALID).  The kernel runs as clusters of 2 CTAs: sms is rounded down to whole clusters, at least one, and
 * capped by the clusters that fit on the device at once -- the result must not depend on it.  ctas_out (optional)
 * receives the number of CTAs launched.                                                                           */
int b200rt_debug_gemm(int epi, const uint16_t* a, const uint16_t* w, const float* bias, const float* resid,
                      void* out, int M, int N, int K, int iters, float* ms_out, const float* ln_stats,
                      const float* ln_gamma, const float* ln_beta, float eps, float* stats_out, int sms, int* ctas_out);
/* b200rt_debug_gemm with flags (b200rt_debug_gemm is this with flags = 0).  B200RT_DEBUG_GEMM_LN512: the LayerNorm'd width may
 * also be 512 -- the CLIP text tower's 4-partial epilogues, epi 0 or 3 with N % 256 == 0.                                  */
#define B200RT_DEBUG_GEMM_LN512 1u
int b200rt_debug_gemm_ex(int epi, const uint16_t* a, const uint16_t* w, const float* bias, const float* resid,
                         void* out, int M, int N, int K, int iters, float* ms_out, const float* ln_stats,
                         const float* ln_gamma, const float* ln_beta, float eps, float* stats_out, int sms, int* ctas_out, uint32_t flags);

/* ctx[B*S,H] (fp16 bits) = multi-head attention of `heads` heads of head_dim over qkv[B*S,3H] (fp16 bits), lens[B],
 * H = heads head_dim; (head_dim, heads) is (64, 12), (32, 12) or (64, 16), 0 meaning 64 and 12.  sms as for
 * b200rt_debug_gemm (it also decides whether units are split by query tile).                                        */
int b200rt_debug_attention(const uint16_t* qkv, const int32_t* lens, uint16_t* ctx, int B, int S, int iters,
                           float* ms_out, int sms, int head_dim, int heads);
/* b200rt_debug_attention with flags (b200rt_debug_attention is this with flags = 0).  B200RT_DEBUG_ATTN_CAUSAL: key k is also
 * masked for query row q when k > q (the CLIP text tower's attention); (head_dim, heads) must then be (64, 8).          */
#define B200RT_DEBUG_ATTN_CAUSAL 1u
int b200rt_debug_attention_ex(const uint16_t* qkv, const int32_t* lens, uint16_t* ctx, int B, int S, int iters,
                              float* ms_out, int sms, int head_dim, int heads, uint32_t flags);

/* Row kernels, one launch each behind host buffers.  hi/lo: fp16 bit patterns [rows, W]; stats: [rows][W/128] (sum, M2)
 * float pairs, one per 128-column slice, M2 about the slice's own mean.  W = 768, except for embed and pool_normalize,
 * whose trailing `hidden` sets it: 768, 384 or 1024 (0 = 768), for embed also 512 (the CLIP text tower, with a zero type0),
 * and for clip_text_pool, which is 512 wide.
 *   embed:          x = (word[ids[t]] + type0) + pos[t % S] -> hi = fp16(x), lo = fp16(x - hi), stats of x.
 *                   word [vocab, W], pos [S, W], type0 [W].
 *   vit_embed:      x = pre_layrnorm((t % T == 0 ? cls : patch_out[t]) + pos[t % T]) -> hi, lo, stats of x.
 *   pool_normalize: out[i] = L2-normalise(LayerNorm(hi + lo of row i * S)), out fp32 [n_items, W].
 *   mean_pool_normalize: out[i] = L2-normalise((1 / L) sum_{r < L} LayerNorm(hi + lo of row i * S + r)), L = lens[i] clamped
 *                   to [1, S] on the device (lens is passed through unchecked); rows past L are never read.  out fp32
 *                   [n_items, W]; W from the trailing `hidden` as for pool_normalize.
 *   vit_pool:       out[i] = L2-normalise(proj . LayerNorm(hi + lo of row i * T)), proj fp32 [P, 768], 1 <= P <= 1024,
 *                   out fp32 [n_items, P].
 *   clip_text_pool: out[i] = L2-normalise(proj . LayerNorm(hi + lo of row i * S + p_i)), p_i the pooled position of item i
 *                   chosen from ids[i * S .. + L) (L = lens[i] clamped to [1, S] on the device; ids past L are never read):
 *                   eos_id == 2, the first position of the largest id; otherwise the first position equal to eos_id, 0
 *                   when there is none.  ids int32 [n_items * S], proj fp32 [P, 512], 1 <= P <= 1024, out fp32 [n_items, P].
 *   fold_ln:        w_out = fp16(w o gamma - rowmean(w o gamma)), cvec_out = w beta + bias (bias may be NULL);
 *                   gamma NULL: w_out = fp16(w) and cvec_out is not written.  w fp32 [N, K], K % 64 == 0.    */
int b200rt_debug_embed(const int32_t* ids, const float* word, const float* pos, const float* type0, int n_tokens, int S, int vocab,
                       uint16_t* hi_out, uint16_t* lo_out, float* stats_out, int hidden);
/*   embed_segs:     embed with token types: token t takes type row 1 when t % S >= segs[t / S] (clamped to [0, S] on the device),
 *                   else row 0.  type [2, W], segs [n_tokens / S], n_tokens a multiple of S; W = hidden (768, 384 or 1024).
 *   cls_head:       out[i] = cls_w . tanh(pool_w . LayerNorm(hi + lo of row i * S) + pool_b) + cls_b, raw logits, out fp32
 *                   [n_items, L], 1 <= L <= 64; pool_w fp32 [W, W], cls_w [L, W], cls_b [L]; W = hidden (768, 384 or 1024).
 *                   ctas: the most blocks launched (0 = one per item); the result must not depend on it.                  */
int b200rt_debug_embed_segs(const int32_t* ids, const int32_t* segs, const float* word, const float* pos, const float* type, int n_tokens,
                            int S, int vocab, uint16_t* hi_out, uint16_t* lo_out, float* stats_out, int hidden);
int b200rt_debug_cls_head(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, const float* pool_w,
                          const float* pool_b, const float* cls_w, const float* cls_b, int n_items, int S, int L, float eps, float* out,
                          int hidden, int ctas);
/*   gemm_splade:    the SPLADE decoder GEMM (EPI_SPLADE_MAX): vmax_out[i, n] = fp32 bits of max(0, max over rows r = i S + t,
 *                   t < lens[i] (clamped to [0, S]), of rstd_r (a_r . w_n) + c[n]) for n < vocab, 0 for n >= vocab.  a fp16
 *                   [B S, K], w fp16 [vocab, K] (rows past vocab read as zeros), c fp32 [N], stats (sum, M2) [B S, K / 128],
 *                   vmax_out uint32 [B, N]; K = 768, 384 or 1024, N % 256 == 0, S % 64 == 0.  iters launches are timed into ms_out
 *                   (optional); the maxima come from one more launch on a zeroed buffer.  sms and ctas_out (optional, the CTAs
 *                   of that launch) as for b200rt_debug_gemm: the result must not depend on sms.
 *   mlm_ln_stats:   stats_out [n_rows, hidden / 128] (sum, M2) partials of the fp16 rows u [n_rows, hidden]; vmax_out [n_max]
 *                   is poisoned (0xFF) and comes back as the kernel leaves it (zeroed).
 *   splade_finalize: out[i, v] = log1p(fp32 bits vmax[i, v]) for v < vocab, vmax uint32 [n_items, vpad], out [n_items, vocab]. */
int b200rt_debug_gemm_splade(const uint16_t* a, const uint16_t* w, const float* c, const float* stats, const int32_t* lens, int B, int S,
                             int N, int K, int vocab, float eps, int sms, int iters, float* ms_out, uint32_t* vmax_out, int* ctas_out);
/* nomic-bert kernels (kernels.h: launch_gemm_rope, launch_gemm_swiglu, launch_attention_stream), one launch each behind host
 * buffers.  gemm_rope: a [M,768] fp16, w [N,768] fp16, c [N], stats [M][6] (NULL: plain acc + c), table float (cos, sin) pairs
 * [n_pos][32] with n_pos >= S, S % 64 == 0, rot_cols a multiple of 256 <= N; out fp16 [M, N].  gemm_swiglu: w [N,768] with
 * gate / up rows interleaved in groups of 8, out fp16 [M, N / 2].  attention_stream: qkv fp16 [B*S, 2304], 64 <= S <= 8192,
 * S % 64 == 0, ctx fp16 [B*S, 768]; ms_out (may be NULL) the mean time of `iters` further launches.  sms: the most CTAs of
 * the persistent launch (0 = every SM); for the two GEMMs, as for b200rt_debug_gemm, with ctas_out (optional) receiving
 * the number of CTAs launched.                                                                                             */
int b200rt_debug_gemm_rope(const uint16_t* a, const uint16_t* w, const float* c, const float* stats, const float* table, int n_pos, int M,
                           int N, int S, int rot_cols, float eps, int sms, uint16_t* out, int* ctas_out);
int b200rt_debug_gemm_swiglu(const uint16_t* a, const uint16_t* w, const float* c, const float* stats, int M, int N, float eps, int sms,
                             uint16_t* out, int* ctas_out);
int b200rt_debug_attention_stream(const uint16_t* qkv, const int32_t* lens, int B, int S, uint16_t* ctx, int sms, int iters, float* ms_out);
int b200rt_debug_mlm_ln_stats(const uint16_t* u, int n_rows, int hidden, size_t n_max, uint32_t* vmax_out, float* stats_out);
int b200rt_debug_splade_finalize(const uint32_t* vmax, int n_items, int vpad, int vocab, float* out);
int b200rt_debug_vit_embed(const uint16_t* patch_out, const float* cls, const float* pos, const float* gamma, const float* beta,
                           int n_rows, int T, float eps, uint16_t* hi_out, uint16_t* lo_out, float* stats_out);
int b200rt_debug_pool_normalize(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, int n_items, int S,
                                float eps, float* out, int hidden);
int b200rt_debug_mean_pool_normalize(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, const int32_t* lens,
                                     int n_items, int S, float eps, float* out, int hidden);
int b200rt_debug_vit_pool(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, const float* proj, int n_items,
                          int T, int P, float eps, float* out);
int b200rt_debug_clip_text_pool(const uint16_t* hi, const uint16_t* lo, const int32_t* ids, const int32_t* lens, const float* gamma,
                                const float* beta, const float* proj, int n_items, int S, int P, float eps, int eos_id, float* out);
int b200rt_debug_fold_ln(const float* w, const float* gamma, const float* beta, const float* bias, int N, int K, uint16_t* w_out,
                         float* cvec_out);

/* Trace of the product forward on replica 0: the workspace is set to 0xFF bytes (NaN in fp16 and fp32), then the first
 * n_launches launches of the forward of this batch run exactly as the product enqueues them (same kernels, buffers and stream,
 * no sync or copy between them), and the workspace is copied out once they finish.  n_launches is in [0, n_total], n_total =
 * 5 layers + 2 (text: embed, 5 per layer, pool_normalize -- mean_pool_normalize for a B200RT_LOAD_POOL_MEAN model,
 * clip_text_pool for kind "clip_text") or 5 layers + 4 (vit: im2col, gemm_patch, vit_embed, 5 per layer, vit_pool), or 5 layers + 5
 * for kind "bert_splade" (embed, 5 per layer, gemm_mlm_transform writing u [M, H] into ctx, mlm_ln_stats writing u's partials
 * into pstats1 and zeroing the uint32 [n_items, vpad] maxima at the start of ffn, gemm_splade raising them, splade_finalize
 * writing out [n_items, vocab]; vpad = vocab rounded up to 256).  Kind "nomic_bert" runs embed, then per layer gemm_qkv_rope,
 * attention_stream, gemm_attn_out, gemm_ffn1_swiglu (silu(g) u [M, I] into ffn), gemm_ffn2, then the pool: 5 layers + 2.
 * max_len may be up to the longest wave the model runs (kind "clip_text": 128, its bucket for items of 65-77 tokens; the
 * lengths stay <= max_pos; kind "nomic_bert": max_pos rounded up to 64, a multiple of 64), as for b200rt_debug_profile_forward.  Every buffer comes back for rows = min(M + 256, R) rows, R = b200rt_debug_model_cap_rows(model) (512
 * b200rt_wave_capacity_items(), or 3/4 of that rounded down to 128 for bge-large), M = n_items * max_len
 * (text) or n_items * tokens (vit), at the model's widths (H = hidden, I = inter, P = H / 128):
 *   yhi, ylo, ctx: fp16 bits [rows, H]; qkv: fp16 bits [rows, 3H]; ffn: fp16 bits [rows, I] (vit: the im2col matrix
 *   [M, 3 p p] is its start until FFN1 overwrites it); pstats0, pstats1: (sum, M2) float pairs [rows, P];
 *   out: fp32 [n_items, out_dim], poisoned too, written by the pool launch.
 * names_out receives the names of the launches run, NUL-terminated and packed (up to names_cap bytes); n_total (optional)
 * the launch count of the whole forward.                                                                                 */
int b200rt_debug_forward_trace(int model, const int32_t* ids, const int32_t* lens, int n_items, int max_len, int n_launches,
                               uint16_t* yhi, uint16_t* ylo, float* pstats0, float* pstats1, uint16_t* qkv, uint16_t* ctx,
                               uint16_t* ffn, float* out, char* names_out, size_t names_cap, int* n_total);
/* b200rt_debug_forward_trace of a sentence-pair batch: segs [n_items] as for b200rt_submit_pairs (classifier models; NULL: one
 * segment).  The last launch of a "bert_classifier" model is "cls_head", which writes out [n_items, num_labels].            */
int b200rt_debug_forward_trace_segs(int model, const int32_t* ids, const int32_t* lens, const int32_t* segs, int n_items, int max_len,
                                    int n_launches, uint16_t* yhi, uint16_t* ylo, float* pstats0, float* pstats1, uint16_t* qkv,
                                    uint16_t* ctx, uint16_t* ffn, float* out, char* names_out, size_t names_cap, int* n_total);
int b200rt_debug_vit_forward_trace(int model, const float* pixels, int n_items, int n_launches, uint16_t* yhi, uint16_t* ylo,
                                   float* pstats0, float* pstats1, uint16_t* qkv, uint16_t* ctx, uint16_t* ffn, float* out,
                                   char* names_out, size_t names_cap, int* n_total);

/* Rows of this model that one replica's workspace holds, the bound of its waves and of a trace: 512
 * b200rt_wave_capacity_items() for bge-base, bge-small and vit; cap_rows * 768 / hidden rounded down to 128 for a wider
 * model (bge-large: 3/4).                                                                                            */
int b200rt_debug_model_cap_rows(int model);

/* Per-kernel device times (ms, CUDA events on the compute stream) of one forward of a resident batch:
 * names_out receives up to cap NUL-terminated names packed in a char buffer, ms_out the times.        */
int b200rt_debug_profile_forward(int model, int n_items, int max_len, int iters, char* names_out, size_t names_cap,
                                 float* ms_out, int* n_out, int cap);

#ifdef __cplusplus
}
#endif
#endif
