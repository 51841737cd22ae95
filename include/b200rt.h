/* b200rt -- C ABI of the in-box H100 runtime behind the `modal` shim's .map() fan-out.
 *
 * The reference (modal-labs/modal-examples) has no native interface for this path: its fan-out is
 *   Function.map  -> cloudpickle -> gRPC -> one container per input -> gather
 * as used at 06_gpu_and_ml/embeddings/text_embeddings_inference.py:167 (`model.embed.map(...)`), and its
 * arithmetic is an HTTP call into an un-vendored TEI server (`POST /embed`, same file :100).  The entry
 * points below are what a binding for that path replaces; each cites the reference interface it stands
 * in for.  Plain pointers and sizes only; every function is thread-safe (forwards on one replica execute one
 * after the other on the device whichever stream they were enqueued on); nothing calls back into the caller.  Return 0 on success, a negative B200RT_E_* code on failure (text via b200rt_last_error()).
 */
#ifndef B200RT_H
#define B200RT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200RT_OK 0
#define B200RT_TIMEOUT 1        /* b200rt_wait: not complete within timeout_ms; b200rt_poll_any: none ready */
#define B200RT_E_INVALID (-1)   /* bad argument (shape, id out of vocabulary, unknown handle) */
#define B200RT_E_STATE (-2)     /* not initialised / already initialised / shut down */
#define B200RT_E_CUDA (-3)      /* CUDA error; the context is poisoned and every later call fails fast */
#define B200RT_E_NOMEM (-4)
#define B200RT_E_UNSUPPORTED (-5) /* e.g. device is not sm_90, or geometry is none the kernels cover */

/* Geometry of a BERT encoder (HF BertConfig fields).  The sm_90a kernels cover three geometries: bge-base (hidden 768,
 * 12 heads of 64, inter 3072), bge-small (hidden 384, 12 heads of 32, inter 1536) and bge-large (hidden 1024, 16 heads of
 * 64, inter 4096), with max_pos <= 512; `layers` is free.  A model's results are `hidden` floats per item.  The workspace
 * is sized for bge-base, so a bge-large wave holds 3/4 of the tokens (b200rt_model_wave_capacity_items); loading a
 * bge-large model returns B200RT_E_INVALID when that is less than one 512-token item.                                */
typedef struct b200rt_bert_config {
    int32_t vocab, hidden, layers, heads, inter, max_pos, type_vocab;
    float eps;
} b200rt_bert_config;

/* A BERT cross-encoder / sequence classifier (HF BertForSequenceClassification): the encoder of `bert` -- one of the three
 * geometries above, type_vocab == 2 -- then BertPooler (dense [hidden, hidden] + tanh on the final LayerNorm of the [CLS] row)
 * and the classifier [num_labels, hidden], 1 <= num_labels <= 64.  Results are num_labels raw logits per item (no sigmoid or
 * softmax: the caller applies them), e.g. cross-encoder/ms-marco-MiniLM-L-6-v2's relevance logit (num_labels = 1), which
 * TEI serves through POST /rerank.                                                                                      */
typedef struct b200rt_bert_classifier_config {
    b200rt_bert_config bert;
    int32_t num_labels;
} b200rt_bert_classifier_config;

/* A nomic-bert encoder (HF NomicBertModel, e.g. nomic-ai/nomic-embed-text-v1 / -v1.5): bge-base's geometry and post-LN
 * layers (bert.hidden 768, 12 heads of 64, inter 3072), with rotary position embeddings on Q and K (rotate_half pairs
 * (d, d + 32) of each head, inv_freq_i = 1 / rope_theta^(i / 32)) instead of a position table, a SwiGLU MLP
 * down(silu(gate(x)) * up(x)), and no biases.  Inputs up to bert.max_pos <= 8192 tokens; layers, vocab and type_vocab >= 1
 * are free (every token takes type row 0).  Results are 768 floats per item.                                             */
typedef struct b200rt_nomic_bert_config {
    b200rt_bert_config bert;
    float rope_theta;
} b200rt_nomic_bert_config;

/* Geometry of a CLIP-style ViT image tower (HF CLIPVisionConfig fields + projection_dim).  The kernels are specialised for
 * ViT-B/16: hidden 768, 12 heads of 64, inter 3072, (image/patch)^2 + 1 <= 512 tokens, 3*patch*patch a multiple of 64. */
typedef struct b200rt_vit_config {
    int32_t image, patch, hidden, layers, heads, inter, proj;
    float eps;
} b200rt_vit_config;

/* Geometry of a CLIP text tower (HF CLIPTextConfig fields + projection_dim + eos_token_id): the text half of the CLIP model
 * the reference's image example serves (image_embeddings_infinity.py:298-306, where infinity's `engine.embed(sentences=...)`
 * runs it).  The kernels cover the tower of openai/clip-vit-base-patch16 (and -patch32): hidden 512, 8 heads of 64, inter
 * 2048, max_pos <= 128 (77 in the checkpoint), proj <= 1024; `layers` and `vocab` are free.  Causal self-attention, pre-LN
 * layers with quick-GELU MLPs; the pooled row of item i is chosen from its ids: eos_id == 2 (HF's legacy branch, the original
 * openai configs) the first position of the largest id, otherwise the first position equal to eos_id (0 when there is none);
 * then final_layer_norm, text_projection [proj, hidden] (no bias) and L2 normalisation.  Results are `proj` floats per item. */
typedef struct b200rt_clip_text_config {
    int32_t vocab, hidden, layers, heads, inter, max_pos, proj, eos_id;
    float eps;
} b200rt_clip_text_config;

typedef struct b200rt_stats_t {
    uint64_t items, waves, tickets;     /* completed so far */
    uint64_t kernel_launches;           /* of this library's own kernels */
    uint64_t h2d_bytes, d2h_bytes;      /* through submit()/wait() */
    uint64_t peer_bytes;                /* scatter + fused-gather bytes that crossed NVLink */
    double stage_us, h2d_scatter_us, forward_us, d2h_us; /* summed per-wave stage times (device events; forward = root replica) */
    double gap_us;                      /* idle time of the first participating replica's compute stream between consecutive waves */
    double dispatch_us;                 /* host time the dispatcher spent forming, staging and enqueueing waves */
    double forward_max_us;              /* summed per wave: the slowest participating replica's forward (device events) */
    double gap_max_us;                  /* summed per wave: the largest idle time any participating replica's compute stream had before it */
} b200rt_stats_t;

/* Replica pool.  Stands in for `@app.cls(gpu=..., max_containers=N)` + `@modal.concurrent`
 * (text_embeddings_inference.py:79-86): n_gpus local H100s instead of N cloud containers.  Enables peer
 * access between all of them and starts the scheduler threads.  devices = NULL means 0..n_gpus-1.    */
/* flags: bits 0-15 = items of 512 tokens one replica takes per wave (0 = default: the SM count of the first device, 132 on an H100 SXM), see B200RT_INIT_WAVE_ITEMS */
#define B200RT_INIT_WAVE_ITEMS(n) ((uint32_t)(n) & 0xFFFFu)
/*        bits 16-23 = k > 0: TWO replicas per GPU; each replica's GEMM launches ask for (SMs - k) SMs and its attention launches
 *        for k, so that one replica's attention (MUFU-bound, light on L2) runs beside the other's GEMMs (L2-fill-bound).       */
#define B200RT_INIT_SPLIT_SMS(k) (((uint32_t)(k) & 0xFFu) << 16)
int b200rt_init(int n_gpus, uint32_t flags);
int b200rt_init_devices(const int* devices, int n_gpus, uint32_t flags);
int b200rt_num_gpus(void);

/* Cold start.  Stands in for `download_model` / `spawn_server` (text_embeddings_inference.py:37-56):
 * one host->root-GPU copy of the fp32 weight blob, fp16 conversion on the GPU, then a peer broadcast
 * over NVLink to the other replicas.  kind = "bert" (cfg: b200rt_bert_config; blob order: b200rt.weights.blob_layout),
 * "vit" (cfg: b200rt_vit_config; the CLIP ViT-B/16 image tower behind 06_gpu_and_ml/embeddings/image_embeddings_infinity.py:76-77;
 * blob order: b200rt.weights.vit_blob_layout) or "clip_text" (cfg: b200rt_clip_text_config; the same model's text tower, which
 * infinity's `embed(sentences=...)` runs -- image_embeddings_infinity.py:298-306; blob order:
 * b200rt.weights.clip_text_blob_layout) or "bert_classifier" (cfg: b200rt_bert_classifier_config; blob order:
 * b200rt.weights.classifier_blob_layout -- BERT's, then pool.w [H,H] | pool.b [H] | cls.w [L,H] | cls.b padded to 128 floats).
 * kind "bert_splade" (cfg: b200rt_bert_config, one of the three geometries, vocab <= 49152 else B200RT_E_UNSUPPORTED) is a
 * SPLADE sparse encoder (HF BertForMaskedLM + SpladePooling(max, relu), e.g. naver/splade-v3): results are vocab floats per item,
 * out[i, v] = log(1 + max over the item's tokens of relu(MLM logit v)); blob order b200rt.weights.splade_blob_layout -- BERT's,
 * then mlm.t.w [H,H] | mlm.t.b [H] | mlm.ln.g [H] | mlm.ln.b [H] | mlm.dec.w [vocab,H] | mlm.dec.b padded to a multiple of 128
 * floats.  It takes b200rt_submit[_ex] and b200rt_embed_device (max_len a multiple of 64); segs are B200RT_E_INVALID.
 * kind "nomic_bert" (cfg: b200rt_nomic_bert_config) is a long-context text encoder: blob order b200rt.weights.nomic_blob_layout
 * -- word [V,H] | type [T,H] | emb.ln.g | emb.ln.b, then per layer qkv.w [3H,H] | ao.w [H,H] | ln1.g | ln1.b | gate.w [I,H] |
 * up.w [I,H] | down.w [H,I] | ln2.g | ln2.b, no biases.  It takes b200rt_submit[_ex] with max_len <= max_pos (items travel in
 * 64-token buckets up to max_pos rounded up to 64: a wave holds 8 items of 8192 tokens on an H100 SXM) and b200rt_embed_device
 * (max_len a multiple of 64, up to max_pos rounded up to 64); segs are B200RT_E_INVALID.
 * A "clip_text" model takes token ids through b200rt_submit[_ex] (max_len <= max_pos,
 * ids < vocab; items travel in the 64- or 128-token bucket) and b200rt_embed_device (max_len <= 128, the longest wave the
 * scheduler forms for it: device-resident callers can run the bucket the scheduler would), and is refused by
 * b200rt_submit_pixels.                                                                                              */
int b200rt_model_load(const char* kind, const void* cfg, const void* weights, size_t nbytes, int* model_out);
/* b200rt_model_load with load flags (b200rt_model_load is this with flags = 0).  B200RT_LOAD_POOL_MEAN (kinds "bert" and
 * "nomic_bert"):
 * pool each item as sentence-transformers' Pooling(mean) + Normalize does -- the mean over the item's lens[i] valid tokens
 * ([CLS] and [SEP] included) of the final hidden states, then L2 normalise -- instead of taking the [CLS] row; the pooling of
 * all-MiniLM-L6-v2, e5, gte and nomic-embed-text.  The forward before the pool, and its launch count, are the same either way.
 * With any other kind, or with any other flag bit set, returns B200RT_E_INVALID.                                                      */
#define B200RT_LOAD_POOL_MEAN 1u
int b200rt_model_load_ex(const char* kind, const void* cfg, const void* weights, size_t nbytes, uint32_t flags, int* model_out);

/* One .map() input.  Stands in for `TextEmbeddingsInference.embed` -> `POST /embed`
 * (text_embeddings_inference.py:97-104) with token ids instead of strings: ids is [n_items, max_len]
 * int32 row-major (positions >= lens[i] are ignored; lens == NULL means every item is max_len long),
 * out receives [n_items, hidden] fp32 unit-norm embeddings.  Host buffers; `out` stays caller-owned and
 * must remain valid until the ticket completes; ids/lens may be reused as soon as submit returns.     */
int b200rt_submit(int model, const int32_t* ids, const int32_t* lens, int n_items, int max_len, float* out,
                  uint64_t* ticket_out);
/* Zero-copy variant (host wire format, SURVEY.md section 8 f2).  B200RT_SUBMIT_BORROW_IDS: the caller keeps `ids` valid
 * and unchanged until the ticket completes, and the library does not take a private copy; when `ids` (at the
 * wave's padded length) and/or `out` lie inside a b200rt_alloc_pinned() allocation they are DMA'd from / to where
 * they lie instead of passing through the scheduler's staging buffers.                                          */
#define B200RT_SUBMIT_BORROW_IDS 1u
int b200rt_submit_ex(int model, const int32_t* ids, const int32_t* lens, int n_items, int max_len, float* out,
                     uint32_t flags, uint64_t* ticket_out);
/* One .map() input of the image example (image_embeddings_infinity.py:330-350, `engine.image_embed(images=...)`), with
 * preprocessed pixels instead of image paths: pixels is [n_items, 3, image, image] fp32 (resized / normalised as CLIP's
 * processor does), out receives [n_items, proj] fp32 unit-norm embeddings.  Both stay caller-owned and must remain valid until
 * the ticket completes; each replica pulls its share of the pixels over its own PCIe link (no scatter through the root:
 * an image is 600 KB, not 2 KB).  Pinned memory (b200rt_alloc_pinned) makes the copies asynchronous.  model: kind "vit". */
int b200rt_submit_pixels(int model, const float* pixels, int n_items, float* out, uint64_t* ticket_out);
/* Sentence pairs for a "bert_classifier" model (TEI's POST /rerank and /predict with [text, text] inputs): as b200rt_submit_ex,
 * plus segs [n_items]: item i is [CLS] a [SEP] b [SEP] and its second segment (token type 1) starts at token segs[i],
 * 0 <= segs[i] <= lens[i]; segs == NULL means one segment (all type 0).  out receives [n_items, num_labels] raw logits.  segs
 * for a model of any other kind is B200RT_E_INVALID.  b200rt_submit[_ex] on a classifier model classifies single sequences.  */
int b200rt_submit_pairs(int model, const int32_t* ids, const int32_t* lens, const int32_t* segs, int n_items, int max_len, float* out,
                        uint32_t flags, uint64_t* ticket_out);
/* Completion, ordered (`order_outputs=True`): a ticket being waited on is never handed to b200rt_poll_any ...  */
int b200rt_wait(uint64_t ticket, int timeout_ms); /* timeout_ms < 0: forever */
/* ... and unordered (`order_outputs=False`, text_embeddings_inference.py:167): next finished ticket
 * that nobody has waited on yet; B200RT_TIMEOUT when none is ready within timeout_ms.                 */
int b200rt_poll_any(uint64_t* ticket_out, int timeout_ms);

/* Device-resident variant for callers that already hold the batch in HBM on replica `gpu` (index into
 * the pool): enqueues the forward of one batch on `stream` (a cudaStream_t; NULL = the replica's own
 * compute stream) and returns without synchronising.  n_items * max_len must fit the model's wave capacity
 * (512 b200rt_model_wave_capacity_items(model) tokens, or B200RT_E_INVALID).                           */
int b200rt_embed_device(int model, int gpu, const int32_t* d_ids, const int32_t* d_lens, int n_items, int max_len,
                        float* d_out, void* stream);
/* b200rt_embed_device with device-resident segment starts d_segs [n_items] (classifier models; NULL: one segment; each is
 * clamped to [0, max_len] on the device, not validated).  b200rt_embed_device is this with d_segs = NULL.                */
int b200rt_embed_device_pairs(int model, int gpu, const int32_t* d_ids, const int32_t* d_lens, const int32_t* d_segs, int n_items,
                              int max_len, float* d_out, void* stream);
int b200rt_device_sync(int gpu);
int b200rt_wave_capacity_items(void); /* items of 512 tokens one replica takes per wave (bge-base, bge-small) */
/* items of 512 tokens one replica takes per wave of this model: b200rt_wave_capacity_items() for bge-base and bge-small,
 * 3/4 of it for bge-large (the rows of a 1024-wide model that the workspace holds, rounded down to 128: 99 on an H100 SXM);
 * images per wave for kind "vit".                                                                                         */
int b200rt_model_wave_capacity_items(int model);

void* b200rt_alloc_pinned(size_t nbytes);
void b200rt_free_pinned(void* p);

int b200rt_stats(b200rt_stats_t* out);
const char* b200rt_last_error(void); /* thread-local */
void b200rt_shutdown(void);

#ifdef __cplusplus
}
#endif
#endif /* B200RT_H */
