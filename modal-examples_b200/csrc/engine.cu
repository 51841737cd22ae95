// b200rt engine: replica pool, cold-start weight broadcast, the per-shard BERT forward, the C++ stream
// scheduler behind Function.map, and the C ABI declared in include/b200rt.h.
//
// Threads: callers (any number, any thread) -> submit queue -> dispatcher (forms waves, stages ids into
// pinned memory, H2D to the root GPU, scatter kernel into peer HBM, enqueues each shard's forward, whose
// last kernel stores straight into the root's gather buffer, then one D2H) -> completer (waits the wave's
// event, hands rows to the tickets' caller-owned buffers, wakes waiters).  No NCCL call and no host
// round-trip between H2D and D2H.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/b200rt.h"
#include "../../include/b200rt_debug.h"
#include "kernels.h"

namespace b200 {
cudaError_t gemm_init_device();
cudaError_t attention_init_device();
cudaError_t kernels_init_device() {
    cudaError_t e = gemm_init_device();
    if (e != cudaSuccess) return e;
    return attention_init_device();
}
}  // namespace b200

using namespace b200;

namespace {

// ------------------------------------------------------------------------------------------ errors

thread_local std::string t_last_error;
std::atomic<bool> g_poisoned{false};

int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    t_last_error = buf;
    if (code == B200RT_E_CUDA) g_poisoned.store(true);
    return code;
}

#define CUDA_TRY(expr)                                                                                      \
    do {                                                                                                    \
        cudaError_t _e = (expr);                                                                            \
        if (_e != cudaSuccess)                                                                              \
            return fail(B200RT_E_CUDA, "%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    } while (0)

// A launch_* call (kernels.h): a launcher refuses operands outside its contract with cudaErrorInvalidValue before any CUDA call,
// and the runtime's own cudaErrorInvalidValue is a non-sticky argument error, so a refusal is the caller's B200RT_E_INVALID and
// leaves the runtime usable; any other error is handled as by CUDA_TRY.
#define LAUNCH_TRY(expr)                                                                                    \
    do {                                                                                                    \
        cudaError_t _e = (expr);                                                                            \
        if (_e == cudaErrorInvalidValue) return fail(B200RT_E_INVALID, "%s refused its operands", #expr);   \
        if (_e != cudaSuccess)                                                                              \
            return fail(B200RT_E_CUDA, "%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    } while (0)

// ------------------------------------------------------------------------------------------ tensor maps

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int load_driver_entry() {
    if (g_encode) return 0;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn)
        return fail(B200RT_E_CUDA, "cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    return 0;
}

// Encoding a map is host work on no context: CUDA_ERROR_INVALID_VALUE means these operands have no map of this layout (a row
// pitch that is not a multiple of 16 bytes, a head too wide for its swizzle), which is the caller's B200RT_E_INVALID.
int map_error(CUresult r) { return r == CUDA_ERROR_INVALID_VALUE ? B200RT_E_INVALID : B200RT_E_CUDA; }

// fp16 2D row-major [rows, cols] -> box {64, box_rows}, 128B swizzle
int make_map_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(map_error(r), "cuTensorMapEncodeTiled(2d %llu x %llu) -> %d",
                                       (unsigned long long)rows, (unsigned long long)cols, (int)r);
    return 0;
}

// fp16 [B, S, width] (qkv: width 3H, ctx: width H, H = 12 head_dim) -> box {head_dim, 128, 1}: one head's 128 rows, 128B
// swizzle for head_dim 64, 64B for head_dim 32 (rows past S are zero-filled on load and clipped on store)
int make_map_qkv(CUtensorMap* m, const void* base, uint64_t B, uint64_t S, uint64_t width, uint32_t head_dim) {
    cuuint64_t dims[3] = {width, S, B};
    cuuint64_t strides[2] = {width * 2, S * width * 2};
    cuuint32_t box[3] = {head_dim, 128, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, head_dim == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(map_error(r), "cuTensorMapEncodeTiled(qkv B=%llu S=%llu) -> %d",
                                       (unsigned long long)B, (unsigned long long)S, (int)r);
    return 0;
}

// ------------------------------------------------------------------------------------------ owned CUDA resources

// One CUDA resource and the device it was made on.  Move-only; it releases the resource on that device when it goes, so a
// runtime, a replica or a model frees what it made on shutdown and on every early return of init or a load alike.  It converts
// to the raw pointer or handle.
template <class H, auto Release>
class Owned {
  public:
    Owned() = default;
    Owned(Owned&& o) noexcept : h_(std::exchange(o.h_, H{})), dev_(o.dev_) {}
    Owned& operator=(Owned&& o) noexcept { std::swap(h_, o.h_); std::swap(dev_, o.dev_); return *this; }
    ~Owned() { reset(); }
    operator H() const { return h_; }
    H get() const { return h_; }
    cudaError_t reset() {  // releases the resource now, and leaves the calling thread on the device it was on
        if (!h_) return cudaSuccess;
        int cur = 0;
        cudaError_t e = cudaGetDevice(&cur);
        if (e == cudaSuccess) e = cudaSetDevice(dev_);
        if (e == cudaSuccess) {
            e = Release(h_);
            cudaSetDevice(cur);
        }
        h_ = H{};
        return e;
    }
  protected:
    template <class Create>
    cudaError_t make(Create create) {  // create(&h) on the current device; on success this holds h instead of what it held
        int dev = 0;
        H h{};
        cudaError_t e = cudaGetDevice(&dev);
        if (e == cudaSuccess) e = create(&h);
        if (e != cudaSuccess) return e;
        reset();
        h_ = h, dev_ = dev;
        return cudaSuccess;
    }
  private:
    H h_{};
    int dev_ = 0;
};

template <class T>
struct DevMem : Owned<T*, cudaFree> {
    cudaError_t alloc(size_t bytes) { return this->make([&](T** p) { return cudaMalloc(p, bytes); }); }
};
template <class T>
struct HostMem : Owned<T*, cudaFreeHost> {  // pinned
    cudaError_t alloc(size_t bytes) { return this->make([&](T** p) { return cudaMallocHost(p, bytes); }); }
};
struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
    cudaError_t create() { return make([](cudaStream_t* s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }); }
};
struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(unsigned flags = cudaEventDefault) { return make([&](cudaEvent_t* e) { return cudaEventCreateWithFlags(e, flags); }); }
};
struct GraphExec : Owned<cudaGraphExec_t, cudaGraphExecDestroy> {
    cudaError_t instantiate(cudaGraph_t g) { return make([&](cudaGraphExec_t* x) { return cudaGraphInstantiate(x, g, 0); }); }
};

// ------------------------------------------------------------------------------------------ model / device state

constexpr int NSLOT = 4;
constexpr int MIN_ITEMS_PER_REPLICA = 8;  // a wave uses fewer replicas rather than giving one fewer items than this
constexpr int MAX_SEQ = 512;
constexpr int MAX_SEQ_LONG = 8192;  // kind "nomic_bert" (streaming attention): max_pos and its longest bucket
constexpr int VIT_WAVE_ITEMS = 64;  // images one replica takes per wave (64 x 197 tokens; 38.5 MB of pixels per wave slot)
constexpr int TEXT_POS_ROWS = 128;  // kind "clip_text": embed_kernel reads pos[t % S] for every row of a wave padded to its bucket

// The text geometries the kernels cover (hidden, heads, inter, causal): bge-base, bge-small and bge-large (kind "bert") and the
// CLIP text tower (kind "clip_text", causal attention).  The ViT tower is bge-base-wide.
struct TextGeometry {
    int hidden, heads, inter;
    bool causal;
};
constexpr int N_TEXT_GEOMETRIES = 4;
constexpr TextGeometry TEXT_GEOMETRIES[N_TEXT_GEOMETRIES] = {
    {768, 12, 3072, false}, {384, 12, 1536, false}, {1024, 16, 4096, false}, {512, 8, 2048, true}};
// index into TEXT_GEOMETRIES of the geometry `hidden` wide (-1: none); the hidden widths are distinct
inline int text_geometry(int hidden) {
    for (int g = 0; g < N_TEXT_GEOMETRIES; ++g)
        if (TEXT_GEOMETRIES[g].hidden == hidden) return g;
    return -1;
}
// Rows of a `hidden`-wide model that the workspace holds: the buffers are sized for bge-base (HIDDEN, QKV_DIM, 3072,
// STAT_PARTS) at the runtime's cap_rows, so a wider model gets cap_rows * 768 / hidden rows, rounded down to a multiple of
// 128 (bge-large: 3/4).  Every width of bge-large is 4/3 of bge-base's, so each of its buffers is then full; bge-base,
// bge-small and the CLIP text tower keep cap_rows.
inline int model_cap_rows(int rt_cap_rows, int hidden) {
    const int64_t r = static_cast<int64_t>(rt_cap_rows) * HIDDEN / hidden;
    return r >= rt_cap_rows ? rt_cap_rows : static_cast<int>(r / 128 * 128);
}

struct LayerW {
    __half *qkv_w, *ao_w, *ff1_w, *ff2_w;
    float *qkv_b, *ao_b, *ln1_g, *ln1_b, *ff1_b, *ff2_b, *ln2_g, *ln2_b;
    // LayerNorm folded into the consuming projections at load time (kernels.h):
    // qkv_w / ff1_w hold fp16(gamma o W, rows centred); *_c = W beta + b
    float *qkv_c, *ff1_c;
    CUtensorMap m_qkv, m_ao, m_ff1, m_ff2;  // box {64,128}: GEMM B operands (two boxes per 256-column tile)
};

struct DevWeights {
    DevMem<float> f32_arena;   // embeddings, biases, LayerNorm params
    DevMem<__half> f16_arena;  // GEMM weights
    float *word = nullptr, *pos = nullptr, *type = nullptr, *emb_g = nullptr, *emb_b = nullptr;
    std::vector<LayerW> layers;
    // ViT (kind "vit"): patch projection (fp16, the stride-p convolution as a [H, 3 p p] matrix), class / position embeddings,
    // pre / post LayerNorm, visual projection; `pos` above holds the position table.  For a ViT layer, LayerW::ln1_* is the
    // LayerNorm folded into QKV and ln2_* the one folded into FFN1 (pre-LN: neither is re-applied to the residual).
    __half* patch_w = nullptr;
    CUtensorMap m_patch;
    float *cls = nullptr, *pre_g = nullptr, *pre_b = nullptr, *post_g = nullptr, *post_b = nullptr, *proj_w = nullptr, *zero_bias = nullptr;
    // CLIP text (kind "clip_text"): word = token_embedding, pos = position_embedding padded to 128 zero rows, type = a zero row,
    // post_g / post_b = final_layer_norm, proj_w = text_projection [proj, hidden]; layers as for ViT (pre-LN).
    // BERT classifier (kind "bert_classifier"): BertPooler dense [H, H] + bias, classifier [L, H] + bias (padded to 128).
    float *pool_w = nullptr, *pool_b = nullptr, *cls_w = nullptr, *cls_b = nullptr;
    // SPLADE (kind "bert_splade"): the MLM head's transform dense (fp16, the last layer's LN2 folded in; mlm_t_c = W beta + b) and
    // decoder (fp16 [vocab, H], its transform LayerNorm folded in, read past vocab as zero rows by TMA; mlm_dec_c [vpad])
    __half *mlm_t_w = nullptr, *mlm_dec_w = nullptr;
    CUtensorMap m_mlm_t, m_mlm_dec;
    float *mlm_t_c = nullptr, *mlm_dec_c = nullptr;
    // nomic-bert (kind "nomic_bert"): pos = 64 zero rows (embed_kernel reads pos[t % 64]), zero_bias the zero bias of every
    // projection, rope the (cos, sin) table [max_pos rounded up to 64][32]; LayerW::ff1_w holds gate and up interleaved
    // (launch_gemm_swiglu) and ff1_c their folded c in the same order
    float* rope = nullptr;  // float2 pairs
};

// The model kinds.  What depends on the kind is answered by one switch without a default below (or in the loaders and the
// forward's head), so that -Wswitch names every place a new kind has to answer.
enum ModelKind { BERT, BERT_CLASSIFIER, BERT_SPLADE, NOMIC_BERT, VIT, CLIP_TEXT };
// in ModelKind order: the name b200rt_model_load_ex takes the kind by, and whether it takes B200RT_LOAD_POOL_MEAN
constexpr struct { const char* name; bool pool_mean_ok; } MODEL_KINDS[] = {
    {"bert", true}, {"bert_classifier", false}, {"bert_splade", false}, {"nomic_bert", true}, {"vit", false}, {"clip_text", false}};
static_assert(sizeof MODEL_KINDS / sizeof MODEL_KINDS[0] == CLIP_TEXT + 1, "one MODEL_KINDS entry per kind");

struct Model {
    ModelKind kind = BERT;
    bool pool_mean = false;  // bert, nomic_bert: mean of the valid tokens' final hidden states (B200RT_LOAD_POOL_MEAN) instead of the CLS row
    int num_labels = 0;      // bert_classifier: the head's L logits per item
    int splade_vpad = 0;     // bert_splade: the vocabulary tiled to a multiple of 256 (results are vocab-wide sparse vectors)
    b200rt_vit_config vcfg{};
    b200rt_clip_text_config tcfg{};
    int vocab = 0, max_pos = 0;  // token-id models (bert, clip_text): the bounds submit checks ids and lengths against
    int hidden = 0, inter = 0, heads = 0, layers = 0;  // encoder geometry, from whichever config the kind has
    int cap_rows = 0;        // rows of this model one replica's workspace holds (model_cap_rows): bounds every wave of it
    float eps = 0.f;
    int tokens = 0;          // vit: (image / patch)^2 + 1
    int out_dim = HIDDEN;    // floats per item in the result
    size_t item_bytes = 0;   // vit: bytes of one item's pixels
    size_t f32_elems = 0, f16_elems = 0;
    std::vector<DevWeights> per_dev;
};

int launches_per_forward(const Model& m) {  // the embedding (vit: 3 launches), 5 per layer, the head (bert_splade: 4)
    switch (m.kind) {
    case BERT: case BERT_CLASSIFIER: case NOMIC_BERT: case CLIP_TEXT: return 1 + 5 * m.layers + 1;
    case BERT_SPLADE: return 1 + 5 * m.layers + 4;
    case VIT: return 3 + 5 * m.layers + 1;
    }
    return 0;
}
int wave_items(const Model& m, int S) {  // items one replica takes in a wave padded to S tokens
    switch (m.kind) { case VIT: return VIT_WAVE_ITEMS; case BERT: case BERT_CLASSIFIER: case BERT_SPLADE: case NOMIC_BERT: case CLIP_TEXT: break; }
    return m.cap_rows / S;
}
bool takes_segments(const Model& m) {  // items carry segment starts (token types of sentence pairs)
    switch (m.kind) { case BERT_CLASSIFIER: return true; case BERT: case BERT_SPLADE: case NOMIC_BERT: case VIT: case CLIP_TEXT: break; }
    return false;
}
bool pads_to_64(const Model& m) {  // padded lengths are multiples of 64 (the SPLADE max epilogue's and streaming attention's blocks)
    switch (m.kind) { case BERT_SPLADE: case NOMIC_BERT: return true; case BERT: case BERT_CLASSIFIER: case VIT: case CLIP_TEXT: break; }
    return false;
}
// The longest padded length a forward runs at: clip_text's waves go up to the 128-token bucket (its position table is padded to
// TEXT_POS_ROWS zero rows), nomic_bert's up to max_pos rounded up to 64 (its rotary table has those rows), the others' max_pos.
int max_wave_len(const Model& m) {
    switch (m.kind) {
    case CLIP_TEXT: return TEXT_POS_ROWS;
    case NOMIC_BERT: return (m.max_pos + 63) / 64 * 64;
    case BERT: case BERT_CLASSIFIER: case BERT_SPLADE: case VIT: break;
    }
    return m.max_pos;
}
// Submit buckets items by length, to multiples of 64 tokens up to this cap; a wave takes one bucket, padded to the bucket size.
int bucket_cap(const Model& m) {
    switch (m.kind) { case NOMIC_BERT: return max_wave_len(m); case BERT: case BERT_CLASSIFIER: case BERT_SPLADE: case VIT: case CLIP_TEXT: break; }
    return MAX_SEQ;
}
// The encoder layers: post-LN (a residual epilogue re-applies the LayerNorm of the rows it adds to) or pre-LN (quick-GELU FFN1),
// causal attention, and rotary: rotary Q / K in the QKV epilogue, the streaming attention kernel and a SwiGLU FFN1.
struct LayerStyle { bool pre_ln, causal, rotary; };
LayerStyle layer_style(const Model& m) {
    switch (m.kind) {
    case BERT: case BERT_CLASSIFIER: case BERT_SPLADE: return {false, false, false};
    case NOMIC_BERT: return {false, false, true};
    case VIT: return {true, false, false};
    case CLIP_TEXT: return {true, true, false};
    }
    return {};
}

// A forward captured as a CUDA graph (see forward), by the model, buffers, stream and shape it was captured with.
struct GraphKey {
    const void *model, *ids, *lens, *out;
    cudaStream_t stream;
    int B, S;
    const void* segs;
    bool operator<(const GraphKey& o) const {
        return std::tie(model, ids, lens, out, stream, B, S, segs) < std::tie(o.model, o.ids, o.lens, o.out, o.stream, o.B, o.S, o.segs);
    }
};
struct GraphEntry {
    GraphExec exec;
    uint64_t launches;
    uint64_t last_use;
};

struct Dev {
    int id = -1;
    int sm_count = 0;
    int sm_gemm = 0, sm_attn = 0;  // SMs a GEMM / an attention launch of this replica asks for (see B200RT_INIT_SPLIT_SMS)
    Stream compute;
    // workspace (capacity cap_rows rows)
    DevMem<__half> yhi, ylo;  // residual stream y = hi + lo, PRE-LayerNorm; hi doubles as the GEMM A operand
    DevMem<float2> pstats[2];  // [rows][STAT_PARTS] (sum, M2) partials: [0] embedding LN / LN2 inputs, [1] LN1 inputs
    DevMem<__half> qkv, ctx, ffn;
    // fp16 [rows, *] box {64,128}: GEMM A operands and the residual stream (res: hi, lo), per TEXT_GEOMETRIES entry, each over
    // that geometry's model_cap_rows rows (a model reads the same buffers densely at its own widths)
    struct ActMaps {
        ResEpi res;  // res.hi doubles as the A operand of QKV and FFN1
        CUtensorMap ctx, ffn;
    } act[N_TEXT_GEOMETRIES];
    std::map<std::pair<int, int>, std::pair<CUtensorMap, CUtensorMap>> m_qkv_by_S;  // (qkv, ctx) 3D maps per (padded length, hidden)
    std::map<std::tuple<const void*, int, int>, OutEpi> m_out_by_M;  // EPI 0/1/3 output maps per (buffer, width, rows): see get_out_maps
    // wave input slots (written by the root's scatter kernel, possibly over NVLink)
    DevMem<int32_t> ids_in[NSLOT], lens_in[NSLOT];
    DevMem<int32_t> segs_in[NSLOT];  // classifier waves' segment starts (allocated when the first classifier model loads)
    DevMem<float> pix_in[NSLOT];     // vit: this replica's share of a wave's pixels (allocated when the first vit model loads)
    Stream copy;                     // vit: H2D of wave k+1's pixels runs here, under the forward of wave k on `compute`
    Event ev_pix[NSLOT];
    DevMem<int32_t> lens_const;      // vit: every item has `tokens` keys
    CUtensorMap m_im2col;            // vit: the ffn buffer viewed as the im2col matrix [rows, 768]
    Event ev_done[NSLOT];
    Event ev_begin[NSLOT], ev_end[NSLOT];  // timing: the forward itself on this replica's compute stream
    int last_slot = -1;                    // completer only: slot of this replica's previous wave (gap statistics)
    std::mutex mu;  // serialises host-side enqueue on this replica (scheduler vs. embed_device/debug)
    // Every forward on this replica uses the same workspace (yhi, ylo, qkv, ctx, ffn, pstats), whichever stream it is
    // enqueued on: ev_ws is recorded behind each forward and waited on ahead of the next one, so forwards from the
    // scheduler's stream and from callers' streams (b200rt_embed_device) execute one after the other on the device.
    Event ev_ws;
    bool ev_ws_armed = false;
    std::map<GraphKey, GraphEntry> graphs;  // cached forwards (see forward); guarded by mu
    uint64_t graph_tick = 0;
    // launcher thread: enqueues this replica's share of a wave (the ~85 launches per replica would otherwise be issued
    // by the one dispatcher thread for all replicas in turn)
    std::thread launcher;
    std::mutex lmu;
    std::condition_variable lcv;
    std::function<void()> ltask;
    bool lstop = false;
};

struct Ticket {
    uint64_t id;
    const Model* mp = nullptr;  // resolved at submit time (the models vector may grow while the ticket is queued)
    std::vector<int32_t> ids;   // private copy [n, S] (empty when the caller lent us its buffer: `borrowed`)
    const int32_t* ids_ext = nullptr;
    const float* pixels = nullptr;  // vit tickets: [n_items, 3, image, image] fp32, caller-owned until completion
    bool borrowed = false, ids_pinned = false, out_pinned = false;
    const int32_t* ids_ptr() const { return borrowed ? ids_ext : ids.data(); }
    std::vector<int32_t> lens;
    std::vector<int32_t> segs;  // segment starts (b200rt_submit_pairs); empty: one segment per item
    int n_items, S;
    float* out;
    // Items travel in length buckets of 64 tokens (each bucket is padded to its own length, not to the input's max_len):
    // `order` lists the item indices sorted by bucket (stable), empty when that is the identity (all items in one bucket).
    std::vector<int32_t> order;
    int item_at(int pos) const { return order.empty() ? pos : order[pos]; }
    std::atomic<int> remaining; // items not yet delivered
    bool done = false;
    int waiters = 0;            // threads blocked in b200rt_wait on this ticket: poll_any must not hand it out
    int status = 0;
    std::string error;
};

// A run of a ticket's items that share a length bucket: positions [begin, begin + count) of the ticket's `order`.
struct Run {
    std::shared_ptr<Ticket> t;
    int begin, count, bucket;
    int next = 0;  // dispatcher cursor within the run
};

struct Segment {
    std::shared_ptr<Ticket> t;
    int ticket_off, count, wave_off;  // ticket_off: position in the ticket's `order`
};

struct Wave {
    int slot;
    int n_items, S;
    int first_dev = 0;        // lowest replica that took part (its events time the forward)
    uint32_t dev_mask = 0;    // replicas that took part
    bool direct_h2d = false;  // some segments were DMA'd from caller-pinned memory
    int out_dim = HIDDEN;     // floats per result row
    std::vector<Segment> segs;
};

struct Runtime {
    std::vector<std::unique_ptr<Dev>> devs;
    int cap_items = 0;   // per replica per wave, at 512 tokens; 0 = one item per SM of the first device (see rt_init)
    int cap_rows = 0;    // cap_items*512 rounded up to 128
    std::vector<std::unique_ptr<Model>> models;
    // root staging per slot
    HostMem<int32_t> h_ids[NSLOT], h_lens[NSLOT];
    HostMem<float> h_out[NSLOT];
    DevMem<int32_t> d_ids_stage[NSLOT], d_lens_stage[NSLOT];
    HostMem<int32_t> h_segs[NSLOT];  // classifier waves only (allocated with the first classifier model)
    DevMem<int32_t> d_segs_stage[NSLOT];
    DevMem<float> d_out_gather[NSLOT];
    Stream s_in, s_out;  // on root
    Event ev_scatter[NSLOT], ev_wave[NSLOT], ev_t0[NSLOT], ev_fwd_end[NSLOT];
    // queues
    std::mutex mu;
    std::condition_variable cv_submit, cv_done, cv_slot, cv_wave, cv_idle;
    std::deque<Run> pending;  // runs in arrival order; a wave takes the front run's bucket and every later run of that bucket
    std::unordered_map<uint64_t, std::shared_ptr<Ticket>> tickets;
    std::deque<uint64_t> finished_unclaimed;
    std::deque<Wave> inflight;
    bool slot_busy[NSLOT] = {};
    int fill_window_us = 200;
    size_t vit_item_bytes = 0;  // bytes of one image of the loaded vit model(s)
    std::chrono::steady_clock::time_point last_submit = std::chrono::steady_clock::now();
    int active_calls = 0;  // threads inside b200rt_wait / b200rt_poll_any (shutdown waits for them to leave)
    uint64_t next_ticket = 1, next_wave = 0;
    bool stopping = false;
    std::thread dispatcher, completer;
    b200rt_stats_t stats{};
    int last_end_slot = -1, last_end_dev = -1;  // completer only
    std::mutex stats_mu;
    std::string async_error;
};

std::mutex g_rt_mu;
Runtime* g_rt = nullptr;

// ------------------------------------------------------------------------------------------ forward

// One forward's input, in the replica's HBM: token ids [B, S] and valid lengths [B] (text), or pixels [B, 3, image, image]
// (vit, S = the model's token count).
struct Input {
    const int32_t* ids;
    const int32_t* lens;
    const float* pixels;
    int B, S;
    const int32_t* segs = nullptr;  // text: per-item segment starts (token types of sentence pairs); NULL: type 0 throughout
};

// A debug view of one forward; the product path passes none.  The forward calls at() ahead of its first launch (name NULL)
// and behind every launch.  The hook keeps the launch names, records a timing event at each call when `timing` is set
// (evs[0] ahead of the first launch, evs[i] behind launch i), and ends the enqueue once `stop_after` launches are in (-1: the
// whole forward).  The events belong to the hook and go with it, whatever the forward returned.
struct LaunchHook {
    int stop_after = -1;
    bool timing = false;
    std::vector<std::string> names;
    std::vector<Event> evs;
    cudaError_t error = cudaSuccess;  // of the first timing event that could not be created or recorded (ends the enqueue)
    bool at(const char* name, cudaStream_t stream) {  // true: enqueue nothing more
        if (name) names.push_back(name);
        if (timing && error == cudaSuccess) {
            evs.emplace_back();
            error = evs.back().create();
            if (error == cudaSuccess) error = cudaEventRecord(evs.back(), stream);
        }
        return error != cudaSuccess || (stop_after >= 0 && names.size() >= static_cast<size_t>(stop_after));
    }
};

int get_qkv_map(Dev& d, const Model& model, int S, const CUtensorMap** out, const CUtensorMap** out_ctx) {
    const int hidden = model.hidden;
    const auto key = std::make_pair(S, hidden);
    auto it = d.m_qkv_by_S.find(key);
    if (it == d.m_qkv_by_S.end()) {
        CUtensorMap m, mc;
        const uint64_t B = static_cast<uint64_t>(model.cap_rows) / S;  // the maps end inside the allocations at any width
        const uint32_t head_dim = hidden / model.heads;
        int rc = make_map_qkv(&m, d.qkv, B, S, 3 * hidden, head_dim);
        if (rc) return rc;
        rc = make_map_qkv(&mc, d.ctx, B, S, hidden, head_dim);
        if (rc) return rc;
        it = d.m_qkv_by_S.emplace(key, std::make_pair(m, mc)).first;
    }
    *out = &it->second.first;
    *out_ctx = &it->second.second;
    return 0;
}

// The output maps of a forward's EPI 0/1/3 GEMMs (kernels.h: {width, M} over the buffer each writes, exactly M rows), made once
// per (buffer, width, M) -- as many as the wave shapes a replica meets -- and kept on the replica.  Making a map is host work:
// forward() makes a forward's maps ahead of a graph capture, as for get_qkv_map.
struct OutMaps {
    const OutEpi *qkv = nullptr, *ffn = nullptr, *ctx = nullptr;  // QKV; GELU / quick-GELU FFN1; ViT patch, SPLADE transform
};
int get_out_maps(Dev& d, const Model& m, int M, OutMaps* om) {
    auto get = [&](const __half* buf, int width, const OutEpi** out) {
        const auto key = std::make_tuple(static_cast<const void*>(buf), width, M);
        auto it = d.m_out_by_M.find(key);
        if (it == d.m_out_by_M.end()) {
            OutEpi oe;
            if (int rc = make_map_2d(&oe.out, buf, M, width, 64)) return rc;
            it = d.m_out_by_M.emplace(key, oe).first;
        }
        *out = &it->second;
        return 0;
    };
    if (!layer_style(m).rotary) {
        if (int rc = get(d.qkv, 3 * m.hidden, &om->qkv)) return rc;
        if (int rc = get(d.ffn, m.inter, &om->ffn)) return rc;
    }
    if (m.kind == VIT || m.kind == BERT_SPLADE)
        if (int rc = get(d.ctx, m.hidden, &om->ctx)) return rc;
    return 0;
}

// Enqueue the forward of one padded batch on `stream` and add the launches it enqueued to `launches`.  out: fp32 [B, out_dim],
// may be peer memory.  Widths, statistic partials and the attention head size follow the model's geometry: three stages, the
// embedding, the encoder layers as the kind's layer_style runs them, and the kind's head.
int forward_enqueue(Dev& d, const Model& m, int dev_index, const Input& in, float* out, cudaStream_t stream, uint64_t& launches,
                    LaunchHook* hook) {
    const DevWeights& w = m.per_dev[dev_index];
    const bool vit = m.kind == VIT;
    const LayerStyle ls = layer_style(m);
    const int B = in.B, S = in.S, M = B * S;
    if (M > m.cap_rows || B > wave_items(m, S))
        return fail(B200RT_E_INVALID, "batch of %d x %d tokens exceeds the model's wave capacity (%d rows)", B, S, m.cap_rows);
    if (pads_to_64(m) && S % 64 != 0)
        return fail(B200RT_E_INVALID, "a %s forward runs at padded lengths that are multiples of 64 (got %d)", MODEL_KINDS[m.kind].name, S);
    const int H = m.hidden, I = m.inter, P = H / 128;
    const Dev::ActMaps& am = d.act[text_geometry(H)];
    const CUtensorMap *mq = nullptr, *mc = nullptr;
    if (int rc = get_qkv_map(d, m, S, &mq, &mc)) return rc;
    OutMaps om;
    if (int rc = get_out_maps(d, m, M, &om)) return rc;
    const int32_t* lens = vit ? d.lens_const : in.lens;
    // residual epilogue: y <- acc + bias + LN(y), LN given by (stats, gamma, beta) -- or + y (pre-LN); new statistics to stats_out
    auto residual = [&](const float* bias, const float2* stats, const float* gamma, const float* beta, float2* stats_out) {
        return ls.pre_ln ? GemmEpi{bias, nullptr, P, nullptr, nullptr, stats_out, m.eps} : GemmEpi{bias, stats, P, gamma, beta, stats_out, m.eps};
    };
    uint64_t nl = 0;
    // counts the launch just enqueued; true once the hook wants no more
    auto step = [&](const char* name) {
        ++nl;
        return hook && hook->at(name, stream);
    };
    auto last = [&](const char* name) {  // the head's last launch
        step(name);
        return 0;
    };
    auto enqueue = [&]() -> int {
        if (hook && hook->at(nullptr, stream)) return 0;
        if (vit) {
            // patches -> im2col rows in the (idle) ffn buffer -> patch projection into the (idle) ctx buffer -> + class / position
            // embeddings, pre_layrnorm -> residual stream + statistics
            const b200rt_vit_config& c = m.vcfg;
            LAUNCH_TRY(launch_im2col(in.pixels, d.ffn, B, c.image, c.patch, stream));
            if (step("im2col")) return 0;
            GemmEpi e_patch{w.zero_bias, nullptr, P, nullptr, nullptr, nullptr, m.eps};
            LAUNCH_TRY(launch_gemm(EPI_BIAS_F16, d.m_im2col, w.m_patch, d.ctx, nullptr, nullptr, om.ctx, e_patch, M, H, 3 * c.patch * c.patch, d.sm_gemm, stream));
            if (step("gemm_patch")) return 0;
            LAUNCH_TRY(launch_vit_embed(d.ctx, w.cls, w.pos, w.pre_g, w.pre_b, d.yhi, d.ylo, d.pstats[0], M, S, m.eps, stream));
            if (step("vit_embed")) return 0;
        } else {
            // clip_text: token + position, its zero type row leaves (word + 0) + pos bit-exact; no embedding LayerNorm
            // nomic_bert: no position table -- pos is 64 zero rows read as pos[t % 64], so the rows are (word + type0) + 0
            LAUNCH_TRY(launch_embed(in.ids, w.word, w.pos, w.type, d.yhi, d.ylo, d.pstats[0], M, m.kind == NOMIC_BERT ? 64 : S, m.vocab, H,
                                  stream, in.segs));
            if (step("embed")) return 0;
        }
        // Post-LN: the embedding LN, then each layer's LN2, folds into QKV and is re-applied by attn-out; LN1 folds into FFN1 and is
        // re-applied by FFN2.  NomicBertModel: h = LN_a(x + o(attn(rope(q), rope(k), v))), y = LN_m(h + down(silu(gate h) up h)).
        const float *prev_g = w.emb_g, *prev_b = w.emb_b;  // post-LN: the LayerNorm that applies to the current residual rows
        for (int l = 0; l < m.layers; ++l) {
            const LayerW& lw = w.layers[l];
            // QKV = LN_prev(y) Wqkv^T + b, the LayerNorm folded into the epilogue
            GemmEpi e_qkv{lw.qkv_c, d.pstats[0], P, nullptr, nullptr, nullptr, m.eps};
            if (ls.rotary) {
                LAUNCH_TRY(launch_gemm_rope(am.res.hi, lw.m_qkv, d.qkv, e_qkv, RopeEpi{reinterpret_cast<const float2*>(w.rope), S, 2 * H}, M, 3 * H, H, d.sm_gemm, stream));
                if (step("gemm_qkv_rope")) return 0;
                LAUNCH_TRY(launch_attention_stream(*mq, d.ctx, lens, B, S, d.sm_attn, stream));
                if (step("attention_stream")) return 0;
            } else {
                LAUNCH_TRY(launch_gemm(EPI_BIAS_F16, am.res.hi, lw.m_qkv, d.qkv, nullptr, nullptr, om.qkv, e_qkv, M, 3 * H, H, d.sm_gemm, stream));
                if (step("gemm_qkv")) return 0;
                LAUNCH_TRY(launch_attention(*mq, *mc, lens, B, S, d.sm_attn, stream, H / m.heads, m.heads, ls.causal));
                if (step("attention")) return 0;
            }
            // y <- ctx Wao^T + b + LN_prev(y) (pre-LN: + y); new row statistics (LN1's) into pstats[1]
            const GemmEpi e_ao = residual(lw.ao_b, d.pstats[0], prev_g, prev_b, d.pstats[1]);
            LAUNCH_TRY(launch_gemm(EPI_BIAS_RES_SPLIT, am.ctx, lw.m_ao, d.yhi, d.ylo, &am.res, nullptr, e_ao, M, H, H, d.sm_gemm, stream));
            if (step("gemm_attn_out")) return 0;
            GemmEpi e_ff1{lw.ff1_c, d.pstats[1], P, nullptr, nullptr, nullptr, m.eps};
            if (ls.rotary) {
                LAUNCH_TRY(launch_gemm_swiglu(am.res.hi, lw.m_ff1, d.ffn, e_ff1, M, 2 * I, H, d.sm_gemm, stream));
                if (step("gemm_ffn1_swiglu")) return 0;
            } else {
                LAUNCH_TRY(launch_gemm(ls.pre_ln ? EPI_BIAS_QGELU_F16 : EPI_BIAS_GELU_F16, am.res.hi, lw.m_ff1, d.ffn, nullptr, nullptr, om.ffn, e_ff1, M, I, H, d.sm_gemm, stream));
                if (step(ls.pre_ln ? "gemm_ffn1_qgelu" : "gemm_ffn1_gelu")) return 0;
            }
            // y <- ffn W2^T + b + LN1(y) (pre-LN: + y); LN2's statistics into pstats[0]
            const GemmEpi e_ff2 = residual(lw.ff2_b, d.pstats[1], lw.ln1_g, lw.ln1_b, d.pstats[0]);
            LAUNCH_TRY(launch_gemm(EPI_BIAS_RES_SPLIT, am.ffn, lw.m_ff2, d.yhi, d.ylo, &am.res, nullptr, e_ff2, M, H, I, d.sm_gemm, stream));
            if (step("gemm_ffn2")) return 0;
            prev_g = lw.ln2_g;
            prev_b = lw.ln2_b;
        }
        switch (m.kind) {
        case BERT_SPLADE: {
            // SPLADE (BertForMaskedLM + max pooling): u = gelu(LN2(y) W_t^T + b_t) into the idle ctx buffer; the partials of u's
            // LayerNorm into the idle pstats[1] and the wave's max buffer (uint32 [B, vpad] in the idle ffn buffer) zeroed; the
            // decoder GEMM max-reduces relu(LN_t(u) W_dec^T + b) over each item's valid tokens into it, and never stores the
            // [M, vocab] logits; log1p once per (item, word) into out
            GemmEpi e_t{w.mlm_t_c, d.pstats[0], P, nullptr, nullptr, nullptr, m.eps};
            LAUNCH_TRY(launch_gemm(EPI_BIAS_GELU_F16, am.res.hi, w.m_mlm_t, d.ctx, nullptr, nullptr, om.ctx, e_t, M, H, H, d.sm_gemm, stream));
            if (step("gemm_mlm_transform")) return 0;
            uint32_t* vmax = reinterpret_cast<uint32_t*>(d.ffn.get());
            LAUNCH_TRY(launch_mlm_ln_stats(d.ctx, d.pstats[1], vmax, M, static_cast<size_t>(B) * m.splade_vpad, H, stream));
            if (step("mlm_ln_stats")) return 0;
            GemmEpi e_dec{w.mlm_dec_c, d.pstats[1], P, nullptr, nullptr, nullptr, m.eps};
            LAUNCH_TRY(launch_gemm_splade(am.ctx, w.m_mlm_dec, e_dec, SpladeEpi{in.lens, S, vmax, m.vocab}, M, m.splade_vpad, H, d.sm_gemm,
                                        stream));
            if (step("gemm_splade")) return 0;
            LAUNCH_TRY(launch_splade_finalize(vmax, out, B, m.splade_vpad, m.vocab, stream));
            return last("splade_finalize");
        }
        case VIT:
            LAUNCH_TRY(launch_vit_pool(d.yhi, d.ylo, w.post_g, w.post_b, w.proj_w, out, B, S, m.vcfg.proj, m.eps, stream));
            return last("vit_pool");
        case CLIP_TEXT:
            LAUNCH_TRY(launch_clip_text_pool(d.yhi, d.ylo, in.ids, in.lens, w.post_g, w.post_b, w.proj_w, out, B, S, m.tcfg.proj, m.eps,
                                           m.tcfg.eos_id, stream));
            return last("clip_text_pool");
        case BERT_CLASSIFIER:
            LAUNCH_TRY(launch_cls_head(d.yhi, d.ylo, prev_g, prev_b, w.pool_w, w.pool_b, w.cls_w, w.cls_b, out, B, S, m.num_labels, m.eps, H,
                                     stream));
            return last("cls_head");
        case BERT: case NOMIC_BERT:
            if (m.pool_mean) {
                LAUNCH_TRY(launch_mean_pool_normalize(d.yhi, d.ylo, prev_g, prev_b, in.lens, out, B, S, m.eps, H, stream));
                return last("mean_pool_normalize");
            }
            LAUNCH_TRY(launch_pool_normalize(d.yhi, d.ylo, prev_g, prev_b, out, B, S, m.eps, H, stream));
            return last("pool_normalize");
        }
        return 0;
    };
    if (int rc = enqueue()) return rc;
    if (hook) CUDA_TRY(hook->error);
    launches += nl;
    return 0;
}

// Small batches are launch-bound (a single 512-token item is ~85 launches of 5-40 us kernels): below
// GRAPH_MAX_ROWS rows the launch sequence is captured once per (buffers, shape) into a CUDA graph and replayed.
// Large waves keep plain launches (their kernels are long enough to hide the launch cost, and graphs per shape would
// only add memory).  The caller holds d.mu.
constexpr int GRAPH_MAX_ROWS = 8192;
constexpr size_t GRAPH_CACHE_MAX = 96;

// The caller holds d.mu.  Orders this forward behind the previous one on the replica's workspace (see Dev::ev_ws) and adds
// its launches to `launches`.  Text batches of at most GRAPH_MAX_ROWS rows without a hook replay their CUDA graph.
int forward(Dev& d, const Model& m, int dev_index, const Input& in, float* out, cudaStream_t stream, uint64_t& launches,
            LaunchHook* hook = nullptr) {
    if (d.ev_ws_armed) CUDA_TRY(cudaStreamWaitEvent(stream, d.ev_ws, 0));
    if (hook || m.kind == VIT || in.B * in.S > GRAPH_MAX_ROWS) {
        if (int rc = forward_enqueue(d, m, dev_index, in, out, stream, launches, hook)) return rc;
    } else {
        const GraphKey key{&m, in.ids, in.lens, out, stream, in.B, in.S, in.segs};
        auto it = d.graphs.find(key);
        if (it == d.graphs.end()) {
            if (d.graphs.size() >= GRAPH_CACHE_MAX) {  // evict the least recently replayed graph
                auto victim = d.graphs.begin();
                for (auto j = d.graphs.begin(); j != d.graphs.end(); ++j)
                    if (j->second.last_use < victim->second.last_use) victim = j;
                d.graphs.erase(victim);
            }
            const CUtensorMap *mq = nullptr, *mc = nullptr;
            if (int rc = get_qkv_map(d, m, in.S, &mq, &mc)) return rc;  // host-side map creation happens outside the capture
            OutMaps om;
            if (int rc = get_out_maps(d, m, in.B * in.S, &om)) return rc;
            uint64_t nl = 0;
            CUDA_TRY(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
            const int rc = forward_enqueue(d, m, dev_index, in, out, stream, nl, nullptr);
            cudaGraph_t graph = nullptr;
            const cudaError_t ce = cudaStreamEndCapture(stream, &graph);
            if (rc) {
                if (graph) cudaGraphDestroy(graph);
                return rc;
            }
            CUDA_TRY(ce);
            GraphEntry ent{{}, nl, 0};
            CUDA_TRY(ent.exec.instantiate(graph));
            cudaGraphDestroy(graph);
            it = d.graphs.emplace(key, std::move(ent)).first;
        }
        it->second.last_use = ++d.graph_tick;
        CUDA_TRY(cudaGraphLaunch(it->second.exec, stream));
        launches += it->second.launches;
    }
    CUDA_TRY(cudaEventRecord(d.ev_ws, stream));
    d.ev_ws_armed = true;
    return 0;
}

// ------------------------------------------------------------------------------------------ scheduler

void finish_ticket_locked(Runtime& rt, const std::shared_ptr<Ticket>& t, int status, const std::string& err) {
    if (t->done) return;
    t->done = true;
    t->status = status;
    t->error = err;
    if (t->waiters == 0) rt.finished_unclaimed.push_back(t->id);  // a blocked b200rt_wait owns the ticket otherwise
    rt.stats.tickets++;
}

void fail_all(Runtime& rt, const std::string& err) {
    std::lock_guard<std::mutex> lk(rt.mu);
    rt.async_error = err;
    for (auto& kv : rt.tickets) finish_ticket_locked(rt, kv.second, B200RT_E_CUDA, err);
    rt.pending.clear();
    rt.cv_done.notify_all();
}

#define SCHED_TRY(expr)                                                                              \
    do {                                                                                             \
        cudaError_t _e = (expr);                                                                     \
        if (_e != cudaSuccess) {                                                                     \
            g_poisoned.store(true);                                                                  \
            fail_all(rt, std::string(#expr) + ": " + cudaGetErrorString(_e));                        \
            return;                                                                                  \
        }                                                                                            \
    } while (0)

// Pinned allocations handed out by b200rt_alloc_pinned: buffers inside one are DMA targets/sources as they are
// (no staging copy through the scheduler's own pinned slots).
std::mutex g_pin_mu;
std::map<uintptr_t, size_t> g_pinned;  // base -> bytes
bool is_pinned(const void* p, size_t nbytes) {
    std::lock_guard<std::mutex> lk(g_pin_mu);
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    auto it = g_pinned.upper_bound(a);
    if (it == g_pinned.begin()) return false;
    --it;
    return a >= it->first && a + nbytes <= it->first + it->second;
}

void launcher_main(Dev* dp) {
    Dev& d = *dp;
    cudaSetDevice(d.id);
    for (;;) {
        std::function<void()> task;
        {
            std::unique_lock<std::mutex> lk(d.lmu);
            d.lcv.wait(lk, [&] { return d.lstop || d.ltask; });
            if (d.lstop && !d.ltask) return;
            task = std::move(d.ltask);
            d.ltask = nullptr;
        }
        task();
    }
}

void dispatcher_main(Runtime* rtp) {
    Runtime& rt = *rtp;
    const int G = static_cast<int>(rt.devs.size());
    Dev& root = *rt.devs[0];
    int rr = 0;  // first replica of the next wave that does not need the whole pool (whole inputs round-robin)
    for (;;) {
        Wave wv;
        {
            std::unique_lock<std::mutex> lk(rt.mu);
            rt.cv_submit.wait(lk, [&] { return rt.stopping || !rt.pending.empty(); });
            if (rt.stopping) return;
            // a free slot
            int slot = static_cast<int>(rt.next_wave % NSLOT);
            rt.cv_slot.wait(lk, [&] { return rt.stopping || !rt.slot_busy[slot]; });
            if (rt.stopping) return;
            if (rt.pending.empty()) continue;
            // Fill policy: a wave that would go out partial waits while submissions keep arriving -- until it is full, or no
            // ticket has arrived for a quiet period (pool busy: 200 us; idle: 40 us, the latency path), or a hard limit
            // (busy 2 ms, idle 1 ms).  A burst of small inputs hitting an idle pool (the start of every .map()) would otherwise
            // go out as a train of fragments, one per free wave slot.
            {
                const int S0 = rt.pending.front().bucket;
                const Model* m0 = rt.pending.front().t->mp;
                const int cap0 = wave_items(*m0, S0) * G;
                auto queued = [&] {
                    int n = 0;
                    for (auto& r : rt.pending)
                        if (r.bucket == S0 && r.t->mp == m0) n += r.count - r.next;
                    return n;
                };
                bool busy = false;
                for (int s2 = 0; s2 < NSLOT; ++s2) busy |= rt.slot_busy[s2];
                const auto quiet = std::chrono::microseconds(busy ? rt.fill_window_us : rt.fill_window_us / 5);
                const auto hard = std::chrono::steady_clock::now() + std::chrono::microseconds(busy ? 10 * rt.fill_window_us : 5 * rt.fill_window_us);
                while (!rt.pending.empty() && queued() < cap0) {
                    const auto now = std::chrono::steady_clock::now();
                    const auto deadline = std::min(hard, rt.last_submit + quiet);
                    if (now >= deadline) break;
                    rt.cv_submit.wait_until(lk, deadline);
                    if (rt.stopping) return;
                }
                if (rt.pending.empty()) continue;
            }
            rt.slot_busy[slot] = true;
            rt.next_wave++;
            wv.slot = slot;
            wv.S = rt.pending.front().bucket;
            wv.n_items = 0;
            const Model* model = rt.pending.front().t->mp;
            // token capacity scales with 512/S: a wave holds the model's cap_rows tokens per replica
            const int cap_items_S = wave_items(*model, wv.S) * G;
            for (auto it = rt.pending.begin(); it != rt.pending.end() && wv.n_items < cap_items_S;) {
                if (it->bucket != wv.S || it->t->mp != model) {
                    ++it;
                    continue;
                }
                const int take = std::min(it->count - it->next, cap_items_S - wv.n_items);
                wv.segs.push_back(Segment{it->t, it->begin + it->next, take, wv.n_items});
                it->next += take;
                wv.n_items += take;
                it = it->next == it->count ? rt.pending.erase(it) : it + 1;
            }
        }
        const int slot = wv.slot, S = wv.S, n = wv.n_items;
        const Model& model = *wv.segs[0].t->mp;
        auto t_host0 = std::chrono::steady_clock::now();
        SCHED_TRY(cudaSetDevice(root.id));
        SCHED_TRY(cudaEventRecord(rt.ev_t0[slot], rt.s_in));
        // Stage the wave's ids on the root GPU.  A segment whose ids the caller lent us in pinned memory, at the
        // wave's own padded length, is DMA'd from where it lies; anything else goes through the slot's pinned buffer
        // (re-strided to the bucket length when the ticket's max_len is shorter).
        const bool vit = model.kind == VIT;
        const int out_dim = model.out_dim;
        bool staged = false;
        auto direct_ids = [&](const Segment& sg) {  // lent, pinned, already at the wave's padded length, items in place
            const Ticket& t = *sg.t;
            return t.borrowed && t.ids_pinned && t.S == S && t.order.empty();
        };
        for (const Segment& sg : wv.segs) {
            if (vit) break;  // image payloads are pulled by each replica itself (below): nothing is staged on the root
            const Ticket& t = *sg.t;
            int32_t* hdst = rt.h_ids[slot] + static_cast<size_t>(sg.wave_off) * S;
            if (direct_ids(sg)) {
                SCHED_TRY(cudaMemcpyAsync(rt.d_ids_stage[slot] + static_cast<size_t>(sg.wave_off) * S,
                                          t.ids_ptr() + static_cast<size_t>(sg.ticket_off) * t.S,
                                          static_cast<size_t>(sg.count) * S * 4, cudaMemcpyHostToDevice, rt.s_in));
                wv.direct_h2d = true;
                continue;
            }
            staged = true;
            if (t.S == S && t.order.empty()) {
                memcpy(hdst, t.ids_ptr() + static_cast<size_t>(sg.ticket_off) * t.S, static_cast<size_t>(sg.count) * S * 4);
            } else {  // re-stride to the bucket length (every item of the run has len <= S), gathering through `order`
                const int ncopy = std::min(t.S, S);
                for (int i = 0; i < sg.count; ++i) {
                    const int32_t* src = t.ids_ptr() + static_cast<size_t>(t.item_at(sg.ticket_off + i)) * t.S;
                    memcpy(hdst + static_cast<size_t>(i) * S, src, static_cast<size_t>(ncopy) * 4);
                    if (S > ncopy) memset(hdst + static_cast<size_t>(i) * S + ncopy, 0, static_cast<size_t>(S - ncopy) * 4);
                }
            }
        }
        if (!vit)
            for (const Segment& sg : wv.segs)
                for (int i = 0; i < sg.count; ++i) rt.h_lens[slot][sg.wave_off + i] = sg.t->lens[sg.t->item_at(sg.ticket_off + i)];
        // a classifier wave carries every item's segment start; an item submitted without one is a single segment (start = len)
        const bool pairs = takes_segments(model);
        if (pairs)
            for (const Segment& sg : wv.segs)
                for (int i = 0; i < sg.count; ++i) {
                    const int it = sg.t->item_at(sg.ticket_off + i);
                    rt.h_segs[slot][sg.wave_off + i] = sg.t->segs.empty() ? sg.t->lens[it] : sg.t->segs[it];
                }
        auto t_host1 = std::chrono::steady_clock::now();
        if (staged) {
            if (!wv.direct_h2d) {
                SCHED_TRY(cudaMemcpyAsync(rt.d_ids_stage[slot], rt.h_ids[slot], static_cast<size_t>(n) * S * 4,
                                          cudaMemcpyHostToDevice, rt.s_in));
            } else {  // mixed wave: only the staged segments come from the slot buffer
                for (const Segment& sg : wv.segs) {
                    if (direct_ids(sg)) continue;
                    SCHED_TRY(cudaMemcpyAsync(rt.d_ids_stage[slot] + static_cast<size_t>(sg.wave_off) * S,
                                              rt.h_ids[slot] + static_cast<size_t>(sg.wave_off) * S,
                                              static_cast<size_t>(sg.count) * S * 4, cudaMemcpyHostToDevice, rt.s_in));
                }
            }
        }
        if (!vit)
            SCHED_TRY(cudaMemcpyAsync(rt.d_lens_stage[slot], rt.h_lens[slot], static_cast<size_t>(n) * 4,
                                      cudaMemcpyHostToDevice, rt.s_in));
        if (pairs)
            SCHED_TRY(cudaMemcpyAsync(rt.d_segs_stage[slot], rt.h_segs[slot], static_cast<size_t>(n) * 4,
                                      cudaMemcpyHostToDevice, rt.s_in));
        // Replicas used by this wave: everyone when there is enough work, otherwise as many as get at least
        // MIN_ITEMS_PER_REPLICA items each, starting from a rotating replica so that consecutive small waves land on
        // different GPUs.  Contiguous item ranges, as even as possible.
        ScatterPlan plan{};
        plan.n_shards = G;
        plan.S = S;
        int used = std::min(G, std::max(1, n / MIN_ITEMS_PER_REPLICA));
        const int first = used == G ? 0 : rr;
        if (used != G) rr = (rr + used) % G;
        const int per = (n + used - 1) / used;
        uint64_t peer_bytes = 0;
        for (int g = 0; g < G; ++g) {
            plan.dst_ids[g] = rt.devs[g]->ids_in[slot];
            plan.dst_lens[g] = rt.devs[g]->lens_in[slot];
            plan.dst_segs[g] = rt.devs[g]->segs_in[slot];
            plan.item_begin[g] = 0;
            plan.item_count[g] = 0;
        }
        for (int k = 0; k < used; ++k) {
            const int g = (first + k) % G;
            const int b0 = std::min(n, k * per), b1 = std::min(n, (k + 1) * per);
            plan.item_begin[g] = b0;
            plan.item_count[g] = b1 - b0;
            if (g != 0) peer_bytes += static_cast<uint64_t>(b1 - b0) * (vit ? out_dim * 4 : S * 4 + 4 + (pairs ? 4 : 0) + out_dim * 4);
        }
        if (!vit) SCHED_TRY(launch_scatter(rt.d_ids_stage[slot], rt.d_lens_stage[slot], plan, rt.s_in, pairs ? rt.d_segs_stage[slot].get() : nullptr));
        SCHED_TRY(cudaEventRecord(rt.ev_scatter[slot], rt.s_in));
        // every participating replica's launcher thread enqueues its own forward (~85 launches each, in parallel)
        std::atomic<uint64_t> launches{1};
        std::atomic<int> left{0};
        std::mutex jm;
        std::condition_variable jcv;
        std::string err;
        int err_code = 0;
        for (int g = 0; g < G; ++g)
            if (plan.item_count[g] > 0) left.fetch_add(1);
        wv.first_dev = -1;
        for (int g = 0; g < G; ++g) {
            if (plan.item_count[g] == 0) continue;
            if (wv.first_dev < 0) wv.first_dev = g;
            wv.dev_mask |= 1u << g;
            Dev& d = *rt.devs[g];
            auto task = [&, g]() {
                Dev& dd = *rt.devs[g];
                std::string e;
                int code = 0;
                auto ck = [&](cudaError_t ce, const char* what) {
                    if (ce != cudaSuccess && e.empty()) { e = std::string(what) + ": " + cudaGetErrorString(ce); code = B200RT_E_CUDA; }
                    return ce == cudaSuccess;
                };
                {
                    std::lock_guard<std::mutex> dl(dd.mu);
                    uint64_t nl = 0;
                    float* dst = rt.d_out_gather[slot] + static_cast<size_t>(plan.item_begin[g]) * out_dim;
                    if (ck(cudaStreamWaitEvent(dd.compute, rt.ev_scatter[slot], 0), "cudaStreamWaitEvent") &&
                        ck(cudaEventRecord(dd.ev_begin[slot], dd.compute), "cudaEventRecord")) {
                        int rc = 0;
                        if (vit) {
                            // this replica's items, segment by segment, straight from the callers' buffers over its own PCIe link
                            const int b0 = plan.item_begin[g], b1 = b0 + plan.item_count[g];
                            for (const Segment& sg : wv.segs) {
                                const int lo = std::max(b0, sg.wave_off), hi = std::min(b1, sg.wave_off + sg.count);
                                if (lo >= hi) continue;
                                const float* src = sg.t->pixels + static_cast<size_t>(sg.ticket_off + (lo - sg.wave_off)) * (model.item_bytes / 4);
                                if (!ck(cudaMemcpyAsync(dd.pix_in[slot] + static_cast<size_t>(lo - b0) * (model.item_bytes / 4), src,
                                                        static_cast<size_t>(hi - lo) * model.item_bytes, cudaMemcpyHostToDevice, dd.copy), "cudaMemcpyAsync(pixels)"))
                                    break;
                            }
                            if (e.empty() && ck(cudaEventRecord(dd.ev_pix[slot], dd.copy), "cudaEventRecord") &&
                                ck(cudaStreamWaitEvent(dd.compute, dd.ev_pix[slot], 0), "cudaStreamWaitEvent"))
                                rc = forward(dd, model, g, Input{nullptr, nullptr, dd.pix_in[slot], plan.item_count[g], model.tokens}, dst,
                                             dd.compute, nl);
                        } else {
                            rc = forward(dd, model, g, Input{dd.ids_in[slot], dd.lens_in[slot], nullptr, plan.item_count[g], S,
                                                             pairs ? dd.segs_in[slot].get() : nullptr}, dst, dd.compute, nl);
                        }
                        if (rc) { e = t_last_error; code = rc; }
                        else {
                            ck(cudaEventRecord(dd.ev_end[slot], dd.compute), "cudaEventRecord");
                            ck(cudaEventRecord(dd.ev_done[slot], dd.compute), "cudaEventRecord");
                        }
                    }
                    launches.fetch_add(nl);
                }
                std::lock_guard<std::mutex> jl(jm);
                if (!e.empty() && err.empty()) { err = e; err_code = code; }
                left.fetch_sub(1);
                jcv.notify_one();
            };
            if (used == 1 && g == 0) {
                task();  // the root's own share of a one-replica wave: no hand-off (latency path)
            } else {
                std::lock_guard<std::mutex> ll(d.lmu);
                d.ltask = task;
                d.lcv.notify_one();
            }
        }
        {
            std::unique_lock<std::mutex> jl(jm);
            jcv.wait(jl, [&] { return left.load() == 0; });
        }
        if (!err.empty()) {
            if (err_code == B200RT_E_CUDA) g_poisoned.store(true);
            fail_all(rt, err);
            return;
        }
        SCHED_TRY(cudaSetDevice(root.id));
        for (int g = 0; g < G; ++g)
            if (plan.item_count[g] > 0) SCHED_TRY(cudaStreamWaitEvent(rt.s_out, rt.devs[g]->ev_done[slot], 0));
        SCHED_TRY(cudaEventRecord(rt.ev_fwd_end[slot], rt.s_out));
        // D2H: rows of a ticket whose `out` lies in pinned memory go straight there; the rest through the slot buffer
        bool any_staged_out = false;
        for (const Segment& sg : wv.segs) {
            if (!(sg.t->out_pinned && sg.t->order.empty())) { any_staged_out = true; continue; }
            SCHED_TRY(cudaMemcpyAsync(sg.t->out + static_cast<size_t>(sg.ticket_off) * out_dim,
                                      rt.d_out_gather[slot] + static_cast<size_t>(sg.wave_off) * out_dim,
                                      static_cast<size_t>(sg.count) * out_dim * 4, cudaMemcpyDeviceToHost, rt.s_out));
        }
        if (any_staged_out)
            SCHED_TRY(cudaMemcpyAsync(rt.h_out[slot], rt.d_out_gather[slot], static_cast<size_t>(n) * out_dim * 4,
                                      cudaMemcpyDeviceToHost, rt.s_out));
        SCHED_TRY(cudaEventRecord(rt.ev_wave[slot], rt.s_out));
        {
            std::lock_guard<std::mutex> sl(rt.stats_mu);
            rt.stats.kernel_launches += launches.load();
            rt.stats.h2d_bytes += vit ? static_cast<uint64_t>(n) * model.item_bytes : static_cast<uint64_t>(n) * (S * 4 + 4 + (pairs ? 4 : 0));
            rt.stats.d2h_bytes += static_cast<uint64_t>(n) * out_dim * 4;
            rt.stats.peer_bytes += peer_bytes;
            rt.stats.stage_us += std::chrono::duration<double, std::micro>(t_host1 - t_host0).count();
            rt.stats.dispatch_us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_host0).count();
        }
        wv.out_dim = out_dim;
        {
            std::lock_guard<std::mutex> lk(rt.mu);
            rt.inflight.push_back(std::move(wv));
            rt.cv_wave.notify_one();
        }
    }
}

void completer_main(Runtime* rtp) {
    Runtime& rt = *rtp;
    cudaSetDevice(rt.devs[0]->id);
    for (;;) {
        Wave wv;
        {
            std::unique_lock<std::mutex> lk(rt.mu);
            rt.cv_wave.wait(lk, [&] { return rt.stopping || !rt.inflight.empty(); });
            if (rt.inflight.empty()) {
                if (rt.stopping) return;
                continue;
            }
            wv = std::move(rt.inflight.front());
            rt.inflight.pop_front();
        }
        const int slot = wv.slot;
        cudaError_t e = cudaEventSynchronize(rt.ev_wave[slot]);
        if (e != cudaSuccess) {
            g_poisoned.store(true);
            fail_all(rt, std::string("wave failed: ") + cudaGetErrorString(e));
            return;
        }
        Dev& fd = *rt.devs[wv.first_dev < 0 ? 0 : wv.first_dev];
        float ms_in = 0, ms_fwd = 0, ms_out = 0;
        cudaEventElapsedTime(&ms_in, rt.ev_t0[slot], rt.ev_scatter[slot]);
        if (cudaEventElapsedTime(&ms_fwd, fd.ev_begin[slot], fd.ev_end[slot]) != cudaSuccess) { ms_fwd = 0; cudaGetLastError(); }
        float ms_gap = 0;
        if (rt.last_end_slot >= 0 && rt.last_end_dev == wv.first_dev &&
            cudaEventElapsedTime(&ms_gap, fd.ev_end[rt.last_end_slot], fd.ev_begin[slot]) != cudaSuccess) {
            ms_gap = 0;
            cudaGetLastError();
        }
        rt.last_end_slot = slot;
        rt.last_end_dev = wv.first_dev;
        cudaEventElapsedTime(&ms_out, rt.ev_fwd_end[slot], rt.ev_wave[slot]);
        float ms_fwd_max = 0, ms_gap_max = 0;  // over the participating replicas (each replica's events on its own device)
        for (size_t g = 0; g < rt.devs.size(); ++g) {
            if (!((wv.dev_mask >> g) & 1)) { rt.devs[g]->last_slot = -1; continue; }
            Dev& dg = *rt.devs[g];
            float f = 0, gp = 0;
            if (cudaEventElapsedTime(&f, dg.ev_begin[slot], dg.ev_end[slot]) != cudaSuccess) { f = 0; cudaGetLastError(); }
            if (dg.last_slot >= 0 && cudaEventElapsedTime(&gp, dg.ev_end[dg.last_slot], dg.ev_begin[slot]) != cudaSuccess) { gp = 0; cudaGetLastError(); }
            dg.last_slot = slot;
            ms_fwd_max = std::max(ms_fwd_max, f);
            ms_gap_max = std::max(ms_gap_max, gp);
        }
        {
            // rows of tickets that already failed or were shut down are not delivered: their owners may have freed `out`
            std::vector<const Segment*> live;
            {
                std::lock_guard<std::mutex> lk(rt.mu);
                for (const Segment& sg : wv.segs)
                    if (!sg.t->done && !(sg.t->out_pinned && sg.t->order.empty())) live.push_back(&sg);
            }
            const size_t od = static_cast<size_t>(wv.out_dim);
            for (const Segment* sg : live) {
                const float* src = rt.h_out[slot] + static_cast<size_t>(sg->wave_off) * od;
                if (sg->t->order.empty()) {
                    memcpy(sg->t->out + static_cast<size_t>(sg->ticket_off) * od, src, static_cast<size_t>(sg->count) * od * 4);
                } else {  // rows go back to the items' own positions
                    for (int i = 0; i < sg->count; ++i)
                        memcpy(sg->t->out + static_cast<size_t>(sg->t->order[sg->ticket_off + i]) * od, src + static_cast<size_t>(i) * od, od * 4);
                }
            }
        }
        {
            std::lock_guard<std::mutex> sl(rt.stats_mu);
            rt.stats.items += wv.n_items;
            rt.stats.waves++;
            rt.stats.h2d_scatter_us += ms_in * 1e3;
            rt.stats.forward_us += ms_fwd * 1e3;
            rt.stats.gap_us += (ms_gap > 0 ? ms_gap : 0) * 1e3;
            rt.stats.d2h_us += ms_out * 1e3;
            rt.stats.forward_max_us += ms_fwd_max * 1e3;
            rt.stats.gap_max_us += ms_gap_max * 1e3;
        }
        {
            std::lock_guard<std::mutex> lk(rt.mu);
            for (const Segment& sg : wv.segs) {
                if (sg.t->remaining.fetch_sub(sg.count) == sg.count) finish_ticket_locked(rt, sg.t, 0, "");
            }
            rt.slot_busy[slot] = false;
            rt.cv_slot.notify_all();
            rt.cv_done.notify_all();
        }
    }
}

// ------------------------------------------------------------------------------------------ init / load

int alloc_dev(Runtime& rt, Dev& d) {
    CUDA_TRY(cudaSetDevice(d.id));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, d.id));
    if (prop.major != 9 || prop.minor != 0)
        return fail(B200RT_E_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", d.id, prop.major, prop.minor);
    d.sm_count = prop.multiProcessorCount;
    if (d.sm_attn >= d.sm_count || d.sm_attn < 2) {  // whole-GPU replica
        d.sm_gemm = d.sm_attn = d.sm_count;
    } else {  // two replicas share this GPU: GEMM launches leave sm_attn SMs to the other replica's attention launches
        d.sm_gemm = d.sm_count - d.sm_attn;
    }
    CUDA_TRY(kernels_init_device());
    CUDA_TRY(d.compute.create());
    CUDA_TRY(d.ev_ws.create(cudaEventDisableTiming));
    const size_t R = rt.cap_rows;
    for (int i = 0; i < 2; ++i) {
        CUDA_TRY(d.pstats[i].alloc(R * STAT_PARTS * sizeof(float2)));
        CUDA_TRY(cudaMemset(d.pstats[i], 0, R * STAT_PARTS * sizeof(float2)));
    }
    CUDA_TRY(d.yhi.alloc(R * HIDDEN * 2));
    CUDA_TRY(d.ylo.alloc(R * HIDDEN * 2));
    CUDA_TRY(d.qkv.alloc(R * QKV_DIM * 2));
    CUDA_TRY(d.ctx.alloc(R * HIDDEN * 2));
    CUDA_TRY(d.ffn.alloc(R * 3072 * 2));
    // padded / stale rows must stay finite (0 * NaN would leak through masked attention probabilities)
    CUDA_TRY(cudaMemset(d.yhi, 0, R * HIDDEN * 2));
    CUDA_TRY(cudaMemset(d.ylo, 0, R * HIDDEN * 2));
    CUDA_TRY(cudaMemset(d.qkv, 0, R * QKV_DIM * 2));
    CUDA_TRY(cudaMemset(d.ctx, 0, R * HIDDEN * 2));
    CUDA_TRY(cudaMemset(d.ffn, 0, R * 3072 * 2));
    for (int g = 0; g < N_TEXT_GEOMETRIES; ++g) {
        const TextGeometry& tg = TEXT_GEOMETRIES[g];
        const size_t rows = model_cap_rows(rt.cap_rows, tg.hidden);
        if (rows < 128) continue;  // no model of this width can be loaded (model_load refuses it)
        if (int rc = make_map_2d(&d.act[g].res.hi, d.yhi, rows, tg.hidden, 128)) return rc;
        if (int rc = make_map_2d(&d.act[g].res.lo, d.ylo, rows, tg.hidden, 128)) return rc;
        if (int rc = make_map_2d(&d.act[g].ctx, d.ctx, rows, tg.hidden, 128)) return rc;
        if (int rc = make_map_2d(&d.act[g].ffn, d.ffn, rows, tg.inter, 128)) return rc;
    }
    for (int s = 0; s < NSLOT; ++s) {
        CUDA_TRY(d.ids_in[s].alloc(R * 4));
        CUDA_TRY(d.lens_in[s].alloc(R * 4));
        CUDA_TRY(cudaMemset(d.ids_in[s], 0, R * 4));
        CUDA_TRY(d.ev_done[s].create(cudaEventDisableTiming));
        CUDA_TRY(d.ev_begin[s].create());
        CUDA_TRY(d.ev_end[s].create());
    }
    return 0;
}

int rt_init(const int* devices, int n, uint32_t flags) {
    std::lock_guard<std::mutex> lk(g_rt_mu);
    if (g_rt) return fail(B200RT_E_STATE, "b200rt already initialised");
    if (g_poisoned.load()) return fail(B200RT_E_CUDA, "context poisoned by an earlier CUDA error");
    if (n < 1 || n > ScatterPlan::MAX_SHARDS) return fail(B200RT_E_INVALID, "n_gpus must be in [1, %d], got %d", ScatterPlan::MAX_SHARDS, n);
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(B200RT_E_CUDA, "no CUDA device available (%s); b200rt has no CPU path", cudaGetErrorString(e));
    auto rt = std::make_unique<Runtime>();
    if (flags & 0xFFFFu) rt->cap_items = static_cast<int>(flags & 0xFFFFu);  // B200RT_INIT_WAVE_ITEMS(n)
    if (rt->cap_items == 0) {
        // Default: as many 512-token items as the GPU has SMs.  A wave of B items is 12B / 36B / 48B GEMM tiles (128 x 256)
        // and 12B attention units, so with B = #SMs every kernel of the forward runs a whole number of rounds
        // (H100 SXM, 132 SMs: 12 / 36 / 48 tiles and 12 attention units per SM).
        int sms = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, devices ? devices[0] : 0) != cudaSuccess || sms < 2) sms = 128;
        rt->cap_items = sms & ~1;
    }
    if (rt->cap_items > 1024) return fail(B200RT_E_INVALID, "wave capacity of %d items per replica is out of range (1..1024)", rt->cap_items);
    rt->cap_rows = ((rt->cap_items * MAX_SEQ + 255) / 256) * 256;
    g_rt = rt.get();  // forward() and friends read capacity through g_rt
    auto bail = [&](int rc) { g_rt = nullptr; return rc; };  // rt goes with the return, and frees what it allocated
    if (int rc = load_driver_entry()) return bail(rc);
    const int split_sms = static_cast<int>((flags >> 16) & 0xFFu);  // B200RT_INIT_SPLIT_SMS(k): two replicas per GPU
    if (split_sms && 2 * n > ScatterPlan::MAX_SHARDS) return bail(fail(B200RT_E_INVALID, "split replicas: at most %d GPUs", ScatterPlan::MAX_SHARDS / 2));
    for (int i = 0; i < n; ++i) {
        for (int half = 0; half < (split_sms ? 2 : 1); ++half) {
            auto d = std::make_unique<Dev>();
            d->id = devices ? devices[i] : i;
            if (d->id < 0 || d->id >= count) return bail(fail(B200RT_E_INVALID, "device %d not present (%d visible)", d->id, count));
            d->sm_attn = split_sms ? split_sms : 1 << 20;
            if (int rc = alloc_dev(*rt, *d)) return bail(rc);
            rt->devs.push_back(std::move(d));
        }
    }
    n = static_cast<int>(rt->devs.size());
    // peer access both ways between every pair (scatter writes root->peer, gather writes peer->root)
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) {
            if (i == j || rt->devs[i]->id == rt->devs[j]->id) continue;
            int can = 0;
            cudaDeviceCanAccessPeer(&can, rt->devs[i]->id, rt->devs[j]->id);
            if (!can) return bail(fail(B200RT_E_UNSUPPORTED, "no peer access between GPU %d and %d", rt->devs[i]->id, rt->devs[j]->id));
            cudaSetDevice(rt->devs[i]->id);
            cudaError_t pe = cudaDeviceEnablePeerAccess(rt->devs[j]->id, 0);
            if (pe == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
            else if (pe != cudaSuccess) return bail(fail(B200RT_E_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(pe)));
        }
    Dev& root = *rt->devs[0];
    if (cudaSetDevice(root.id) != cudaSuccess) return bail(fail(B200RT_E_CUDA, "cudaSetDevice(root)"));
    const size_t wave_rows = static_cast<size_t>(rt->cap_rows) * n;
    auto ck = [&](cudaError_t ce, const char* what) { return ce == cudaSuccess ? 0 : fail(B200RT_E_CUDA, "%s: %s", what, cudaGetErrorString(ce)); };
    if (int rc = ck(rt->s_in.create(), "stream")) return bail(rc);
    if (int rc = ck(rt->s_out.create(), "stream")) return bail(rc);
    for (int s = 0; s < NSLOT; ++s) {
        if (int rc = ck(rt->h_ids[s].alloc(wave_rows * 4), "cudaMallocHost ids")) return bail(rc);
        if (int rc = ck(rt->h_lens[s].alloc(wave_rows * 4), "cudaMallocHost lens")) return bail(rc);
        if (int rc = ck(rt->h_out[s].alloc(wave_rows * HIDDEN * 4), "cudaMallocHost out")) return bail(rc);
        if (int rc = ck(rt->d_ids_stage[s].alloc(wave_rows * 4), "cudaMalloc")) return bail(rc);
        if (int rc = ck(rt->d_lens_stage[s].alloc(wave_rows * 4), "cudaMalloc")) return bail(rc);
        if (int rc = ck(rt->d_out_gather[s].alloc(wave_rows * HIDDEN * 4), "cudaMalloc")) return bail(rc);
        for (Event* ev : {&rt->ev_scatter[s], &rt->ev_wave[s], &rt->ev_t0[s], &rt->ev_fwd_end[s]})
            if (int rc = ck(ev->create(), "cudaEventCreate")) return bail(rc);
    }
    for (auto& d : rt->devs) {
        cudaSetDevice(d->id);
        if (int rc = ck(cudaDeviceSynchronize(), "device sync after init")) return bail(rc);
    }
    for (auto& d : rt->devs) d->launcher = std::thread(launcher_main, d.get());
    rt->dispatcher = std::thread(dispatcher_main, rt.get());
    rt->completer = std::thread(completer_main, rt.get());
    g_rt = rt.release();
    return 0;
}

// ---- weight layouts
//
// A model kind describes its weights as one list: the blob's tensors in blob order, plus arena-only vectors that have no blob
// bytes.  Each entry gives the tensor's size, where it lands in a replica's DevWeights and what the root does with it.
// load_weights walks the list once for every blob offset and arena offset; the root's copies and every replica's pointers
// are both taken from those offsets.

// a DevWeights member (layer < 0) or a member of its layers[layer]
template <class T>
struct Slot {
    using Top = T DevWeights::*;
    using PerLayer = T LayerW::*;
    Top top = nullptr;
    PerLayer per_layer = nullptr;
    T* in(DevWeights& w, int layer) const { return layer >= 0 ? &(w.layers[layer].*per_layer) : top ? &(w.*top) : nullptr; }
};

struct LayoutEntry {
    enum Op {
        COPY,     // fp32 blob tensor, copied
        HALF,     // fp32 blob GEMM weight [n, k] -> fp16, with a LayerNorm folded in when gamma >= 0 (kernels.h)
        ZERO,     // arena only: zero fp32
        DERIVED,  // arena only: the fp32 c = W beta + b that the folding HALF entry naming it writes
    } op;
    size_t n, k;  // n * k elements (fp32 entries: k = 1)
    int layer;
    Slot<float*> f32;
    Slot<__half*> f16;      // HALF: the weight and its GEMM B-operand map (box {64,128})
    Slot<CUtensorMap> map;
    int gamma = -1, beta = -1, bias = -1, cvec = -1;  // a folding HALF: the entries it reads and the DERIVED one it writes
    size_t src = 0, off = 0;  // blob offset, arena offset (set by load_weights)
};

struct Layout {
    std::vector<LayoutEntry> e;
    int add(const LayoutEntry& x) {
        e.push_back(x);
        return static_cast<int>(e.size()) - 1;
    }
    int copy(size_t n, float* DevWeights::*dst) { return add({LayoutEntry::COPY, n, 1, -1, {dst}}); }
    int copy(int l, size_t n, float* LayerW::*dst) { return add({LayoutEntry::COPY, n, 1, l, {nullptr, dst}}); }
    void zero(size_t n, float* DevWeights::*dst = nullptr) { add({LayoutEntry::ZERO, n, 1, -1, {dst}}); }
    int half(size_t n, size_t k, __half* DevWeights::*dst, CUtensorMap DevWeights::*map) {
        return add({LayoutEntry::HALF, n, k, -1, {}, {dst}, {map}});
    }
    int half(int l, size_t n, size_t k, __half* LayerW::*dst, CUtensorMap LayerW::*map) {
        return add({LayoutEntry::HALF, n, k, l, {}, {nullptr, dst}, {nullptr, map}});
    }
    // fold the LayerNorm (entries gamma, beta) into HALF entry w; c = W beta + (entry bias) lands in w's layer's member `c`
    void fold(int w, int gamma, int beta, int bias, float* LayerW::*c) {
        const int cv = add({LayoutEntry::DERIVED, e[w].n, 1, e[w].layer, {nullptr, c}});
        LayoutEntry& x = e[w];
        x.gamma = gamma, x.beta = beta, x.bias = bias, x.cvec = cv;
    }
    // a DevWeights-level HALF entry w: c has c_n >= e[w].n floats, the ones past e[w].n zero
    void fold(int w, int gamma, int beta, int bias, float* DevWeights::*c, size_t c_n) {
        const int cv = add({LayoutEntry::DERIVED, c_n, 1, -1, {c}});
        LayoutEntry& x = e[w];
        x.gamma = gamma, x.beta = beta, x.bias = bias, x.cvec = cv;
    }
};

// a pre-LN layer (ViT, CLIP text): ln1.g ln1.b qkv.w qkv.b ao.w ao.b ln2.g ln2.b ff1.w ff1.b ff2.w ff2.b; QKV folds ln1, FFN1 ln2
void pre_ln_layer(Layout& L, int l, size_t H, size_t I) {
    const int ln1_g = L.copy(l, H, &LayerW::ln1_g), ln1_b = L.copy(l, H, &LayerW::ln1_b);
    const int qkv = L.half(l, 3 * H, H, &LayerW::qkv_w, &LayerW::m_qkv);
    L.fold(qkv, ln1_g, ln1_b, L.copy(l, 3 * H, &LayerW::qkv_b), &LayerW::qkv_c);
    L.half(l, H, H, &LayerW::ao_w, &LayerW::m_ao);
    L.copy(l, H, &LayerW::ao_b);
    const int ln2_g = L.copy(l, H, &LayerW::ln2_g), ln2_b = L.copy(l, H, &LayerW::ln2_b);
    const int ff1 = L.half(l, I, H, &LayerW::ff1_w, &LayerW::m_ff1);
    L.fold(ff1, ln2_g, ln2_b, L.copy(l, I, &LayerW::ff1_b), &LayerW::ff1_c);
    L.half(l, H, I, &LayerW::ff2_w, &LayerW::m_ff2);
    L.copy(l, H, &LayerW::ff2_b);
}

// the fp32 blob onto the root, an fp32 and an fp16 arena (m.f32_elems, m.f16_elems) on every replica; leaves the root current
int upload_blob(Runtime& rt, Model& m, const float* blob, size_t nbytes, DevMem<float>& d_blob) {
    Dev& root = *rt.devs[0];
    CUDA_TRY(cudaSetDevice(root.id));
    CUDA_TRY(d_blob.alloc(nbytes));
    CUDA_TRY(cudaMemcpy(d_blob, blob, nbytes, cudaMemcpyHostToDevice));
    for (size_t g = 0; g < rt.devs.size(); ++g) {
        CUDA_TRY(cudaSetDevice(rt.devs[g]->id));
        CUDA_TRY(m.per_dev[g].f32_arena.alloc(m.f32_elems * 4));
        CUDA_TRY(m.per_dev[g].f16_arena.alloc(m.f16_elems * 2));
    }
    CUDA_TRY(cudaSetDevice(root.id));
    return 0;
}

// once the root's carve (enqueued on its compute stream) is done: free the blob, then the one-time broadcast of the root's
// arenas to the other replicas over NVLink
int broadcast_arenas(Runtime& rt, Model& m, DevMem<float>& d_blob) {
    Dev& root = *rt.devs[0];
    CUDA_TRY(cudaStreamSynchronize(root.compute));
    CUDA_TRY(d_blob.reset());
    for (size_t g = 1; g < rt.devs.size(); ++g) {
        CUDA_TRY(cudaMemcpyPeerAsync(m.per_dev[g].f32_arena, rt.devs[g]->id, m.per_dev[0].f32_arena, root.id, m.f32_elems * 4, root.compute));
        CUDA_TRY(cudaMemcpyPeerAsync(m.per_dev[g].f16_arena, rt.devs[g]->id, m.per_dev[0].f16_arena, root.id, m.f16_elems * 2, root.compute));
    }
    CUDA_TRY(cudaStreamSynchronize(root.compute));
    return 0;
}

// m's weights as L lists them, on every replica: checks the blob's size, has the root carve its arenas out of the blob on the
// GPU (copies, fp16 conversions, LayerNorm folds, zero fills), broadcasts them, and sets every replica's pointers and weight
// tensor maps.  The caller holds the root replica's mu.
int load_weights(Runtime& rt, Model& m, Layout& L, const float* blob, size_t nbytes) {
    size_t blob_elems = 0;
    for (LayoutEntry& e : L.e) {
        // Tensors lie back to back, so each size keeps the next tensor 16-byte aligned: the row kernels read fp32 vectors as
        // float4, the GEMM epilogues as float2, and TMA needs 16-byte fp16 bases.
        if (e.n * e.k % 8 != 0) return fail(B200RT_E_STATE, "internal: a %zu-element weight tensor misaligns the arena", e.n * e.k);
        size_t& arena = e.op == LayoutEntry::HALF ? m.f16_elems : m.f32_elems;
        e.src = blob_elems, e.off = arena;
        arena += e.n * e.k;
        if (e.op == LayoutEntry::COPY || e.op == LayoutEntry::HALF) blob_elems += e.n * e.k;
    }
    if (nbytes != blob_elems * 4) return fail(B200RT_E_INVALID, "weight blob is %zu bytes, geometry needs %zu", nbytes, blob_elems * 4);

    m.per_dev.resize(rt.devs.size());
    Dev& root = *rt.devs[0];
    DevMem<float> d_blob;
    if (int rc = upload_blob(rt, m, blob, nbytes, d_blob)) return rc;
    const DevWeights& rw = m.per_dev[0];
    auto blob_at = [&](int i) -> const float* { return i < 0 ? nullptr : d_blob + L.e[i].src; };
    // a DERIVED entry may be longer than the fold that writes it (the SPLADE decoder's c, padded to its tiles): zeros past it
    CUDA_TRY(cudaMemsetAsync(rw.f32_arena, 0, m.f32_elems * 4, root.compute));
    for (const LayoutEntry& e : L.e) {
        if (e.op == LayoutEntry::COPY)
            CUDA_TRY(cudaMemcpyAsync(rw.f32_arena + e.off, d_blob + e.src, e.n * 4, cudaMemcpyDeviceToDevice, root.compute));
        else if (e.op == LayoutEntry::ZERO)
            CUDA_TRY(cudaMemsetAsync(rw.f32_arena + e.off, 0, e.n * 4, root.compute));
        else if (e.op == LayoutEntry::HALF)
            LAUNCH_TRY(launch_fold_ln(d_blob + e.src, blob_at(e.gamma), blob_at(e.beta), blob_at(e.bias), rw.f16_arena + e.off,
                                    e.cvec < 0 ? nullptr : rw.f32_arena + L.e[e.cvec].off, static_cast<int>(e.n), static_cast<int>(e.k),
                                    root.compute));
    }
    if (int rc = broadcast_arenas(rt, m, d_blob)) return rc;
    for (size_t g = 0; g < rt.devs.size(); ++g) {
        DevWeights& w = m.per_dev[g];
        CUDA_TRY(cudaSetDevice(rt.devs[g]->id));
        w.layers.resize(m.layers);
        for (const LayoutEntry& e : L.e) {
            if (e.op != LayoutEntry::HALF) {
                if (float** p = e.f32.in(w, e.layer)) *p = w.f32_arena + e.off;
                continue;
            }
            __half* q = *e.f16.in(w, e.layer) = w.f16_arena + e.off;
            if (int rc = make_map_2d(e.map.in(w, e.layer), q, e.n, e.k, 128)) return rc;
        }
    }
    return 0;
}

int register_model(Runtime& rt, std::unique_ptr<Model> m, int* model_out) {
    CUDA_TRY(cudaSetDevice(rt.devs[0]->id));
    std::lock_guard<std::mutex> lk(rt.mu);
    rt.models.push_back(std::move(m));
    *model_out = static_cast<int>(rt.models.size()) - 1;
    return 0;
}

// model_load* run under the root replica's mu (b200rt_model_load_ex)

// Segment-start buffers of classifier waves: root staging per slot and every replica's input slots, allocated once, when the
// first classifier model loads (an embedding-only runtime never has them).
int alloc_seg_slots(Runtime& rt) {
    if (rt.h_segs[0]) return 0;
    const size_t wave_rows = static_cast<size_t>(rt.cap_rows) * rt.devs.size();
    for (auto& d : rt.devs) {
        CUDA_TRY(cudaSetDevice(d->id));
        for (int s = 0; s < NSLOT; ++s) CUDA_TRY(d->segs_in[s].alloc(rt.cap_rows * 4));
    }
    CUDA_TRY(cudaSetDevice(rt.devs[0]->id));
    for (int s = 0; s < NSLOT; ++s) {
        CUDA_TRY(rt.d_segs_stage[s].alloc(wave_rows * 4));
        CUDA_TRY(rt.h_segs[s].alloc(wave_rows * 4));
    }
    return 0;
}

constexpr int MAX_LABELS = 64;   // the classifier head's logits per item (launch_cls_head)
constexpr int CLS_B_FLOATS = 128;  // the classifier bias is padded to 128 floats in the blob (tensor sizes keep the arena aligned)
// A SPLADE result is vocab floats per item and an item has at least 64 rows, so vocab <= 64 HIDDEN keeps every wave's results
// inside the gather and pinned staging buffers (HIDDEN floats per row of the wave), and its uint32 [B, vpad] maxima inside the
// ffn buffer (3072 fp16 per row), with no new allocation.
constexpr int SPLADE_MAX_VOCAB = 64 * HIDDEN;
static_assert(static_cast<size_t>((SPLADE_MAX_VOCAB + 255) / 256 * 256) * 4 <= static_cast<size_t>(64) * 3072 * 2, "SPLADE maxima in ffn");

// A model of `kind` with its config's geometry (and token-id bounds), cap_rows rows per wave and out_dim floats per result.
template <class Config>
std::unique_ptr<Model> new_model(ModelKind kind, const Config& c, int cap_rows, int out_dim) {
    auto m = std::make_unique<Model>();
    m->kind = kind, m->hidden = c.hidden, m->inter = c.inter, m->heads = c.heads, m->layers = c.layers, m->eps = c.eps;
    if constexpr (!std::is_same<Config, b200rt_vit_config>::value) m->vocab = c.vocab, m->max_pos = c.max_pos;
    m->cap_rows = cap_rows, m->out_dim = out_dim;
    return m;
}

// Kinds "bert", "bert_classifier" (num_labels: its logits per item) and "bert_splade".  The classifier is the BERT layout
// followed by the pooler and the classifier, with the head as the last launch instead of a pool; the SPLADE encoder is the BERT
// layout followed by BertForMaskedLM's head, with the four SPLADE launches instead of a pool.
int model_load(ModelKind kind, const b200rt_bert_config& c, int num_labels, const float* blob, size_t nbytes, bool pool_mean,
               int* model_out) {
    Runtime& rt = *g_rt;
    if (kind == BERT_CLASSIFIER && (num_labels < 1 || num_labels > MAX_LABELS))
        return fail(B200RT_E_UNSUPPORTED, "num_labels %d outside [1, %d]", num_labels, MAX_LABELS);
    bool known = false;
    for (const TextGeometry& tg : TEXT_GEOMETRIES) known |= !tg.causal && c.hidden == tg.hidden && c.heads == tg.heads && c.inter == tg.inter;
    if (!known || c.max_pos > MAX_SEQ || c.max_pos < 1 || c.layers < 1 || c.vocab < 1 || c.type_vocab < 1)
        return fail(B200RT_E_UNSUPPORTED,
                    "kernels cover three geometries, bge-base (hidden=768 heads=12 inter=3072), bge-small (hidden=384 heads=12 "
                    "inter=1536) and bge-large (hidden=1024 heads=16 inter=4096), with max_pos<=512 (got hidden %d heads %d inter %d "
                    "max_pos %d)", c.hidden, c.heads, c.inter, c.max_pos);
    if (kind == BERT_SPLADE && c.vocab > SPLADE_MAX_VOCAB)
        return fail(B200RT_E_UNSUPPORTED, "a SPLADE vocabulary of %d words exceeds %d (one vocab-wide result per 64 tokens must fit the "
                    "wave's result buffers)", c.vocab, SPLADE_MAX_VOCAB);
    if (kind == BERT_CLASSIFIER && c.type_vocab != 2)
        return fail(B200RT_E_UNSUPPORTED, "a classifier takes sentence pairs through two token types: type_vocab must be 2, got %d",
                    c.type_vocab);
    const int cap_rows = model_cap_rows(rt.cap_rows, c.hidden);
    if (cap_rows < MAX_SEQ)
        return fail(B200RT_E_INVALID,
                    "a hidden=%d model needs room for one %d-token item, and the workspace holds %d of its rows: initialise with a "
                    "larger B200RT_INIT_WAVE_ITEMS (now %d)", c.hidden, MAX_SEQ, cap_rows, rt.cap_items);

    auto m = new_model(kind, c, cap_rows, kind == BERT_CLASSIFIER ? num_labels : kind == BERT_SPLADE ? c.vocab : c.hidden);
    m->pool_mean = pool_mean, m->num_labels = num_labels;  // num_labels: 0 but for a classifier
    if (kind == BERT_SPLADE) m->splade_vpad = (c.vocab + 255) / 256 * 256;

    // b200rt.weights.blob_layout.  QKV of layer l folds the LayerNorm in front of it, the previous layer's ln2 (the embedding
    // LN for l = 0); FFN1 folds the layer's own ln1.
    const size_t H = c.hidden, I = c.inter;
    Layout L;
    L.copy(c.vocab * H, &DevWeights::word);
    L.copy(c.max_pos * H, &DevWeights::pos);
    L.copy(c.type_vocab * H, &DevWeights::type);
    int ln_g = L.copy(H, &DevWeights::emb_g);
    int ln_b = L.copy(H, &DevWeights::emb_b);
    for (int l = 0; l < c.layers; ++l) {
        const int qkv = L.half(l, 3 * H, H, &LayerW::qkv_w, &LayerW::m_qkv);
        L.fold(qkv, ln_g, ln_b, L.copy(l, 3 * H, &LayerW::qkv_b), &LayerW::qkv_c);
        L.half(l, H, H, &LayerW::ao_w, &LayerW::m_ao);
        L.copy(l, H, &LayerW::ao_b);
        const int ln1_g = L.copy(l, H, &LayerW::ln1_g), ln1_b = L.copy(l, H, &LayerW::ln1_b);
        const int ff1 = L.half(l, I, H, &LayerW::ff1_w, &LayerW::m_ff1);
        L.fold(ff1, ln1_g, ln1_b, L.copy(l, I, &LayerW::ff1_b), &LayerW::ff1_c);
        L.half(l, H, I, &LayerW::ff2_w, &LayerW::m_ff2);
        L.copy(l, H, &LayerW::ff2_b);
        ln_g = L.copy(l, H, &LayerW::ln2_g);
        ln_b = L.copy(l, H, &LayerW::ln2_b);
    }
    if (kind == BERT_CLASSIFIER) {  // b200rt.weights.classifier_blob_layout: pool.w [H,H] | pool.b [H] | cls.w [L,H] | cls.b [128]
        L.copy(H * H, &DevWeights::pool_w);
        L.copy(H, &DevWeights::pool_b);
        L.copy(static_cast<size_t>(num_labels) * H, &DevWeights::cls_w);
        L.copy(CLS_B_FLOATS, &DevWeights::cls_b);
        if (int rc = alloc_seg_slots(rt)) return rc;
    }
    if (kind == BERT_SPLADE) {  // b200rt.weights.splade_blob_layout: mlm.t.w [H,H] | mlm.t.b [H] | mlm.ln.g [H] | mlm.ln.b [H] | mlm.dec.w [V,H] | mlm.dec.b
        // [V rounded up to 128]; the transform folds the last layer's LN2, the decoder the transform's LayerNorm
        const int tw = L.half(H, H, &DevWeights::mlm_t_w, &DevWeights::m_mlm_t);
        L.fold(tw, ln_g, ln_b, L.copy(H, nullptr), &DevWeights::mlm_t_c, H);
        const int tg = L.copy(H, nullptr), tb = L.copy(H, nullptr);
        const int dw = L.half(c.vocab, H, &DevWeights::mlm_dec_w, &DevWeights::m_mlm_dec);
        L.fold(dw, tg, tb, L.copy((c.vocab + 127) / 128 * 128, nullptr), &DevWeights::mlm_dec_c, m->splade_vpad);
    }
    if (int rc = load_weights(rt, *m, L, blob, nbytes)) return rc;
    return register_model(rt, std::move(m), model_out);
}

int model_load_vit(const b200rt_vit_config& c, const float* blob, size_t nbytes, int* model_out) {
    Runtime& rt = *g_rt;
    const int grid = c.patch > 0 ? c.image / c.patch : 0;
    const int T = grid * grid + 1;
    const size_t H = HIDDEN, I = 3072, PD = static_cast<size_t>(3) * c.patch * c.patch, P = static_cast<size_t>(c.proj);
    if (c.hidden != HIDDEN || c.heads != HEADS || c.inter != 3072 || c.layers < 1 || c.patch < 2 || c.image % c.patch != 0 || T > MAX_SEQ ||
        PD != HIDDEN || c.patch % 2 != 0 || c.proj < 1 || c.proj > 1024)
        return fail(B200RT_E_UNSUPPORTED, "kernels are specialised for ViT-B: hidden=768 heads=12 inter=3072, <= 512 tokens, 3*patch^2 %% 64 == 0, proj <= 1024 "
                                          "(got hidden %d heads %d inter %d image %d patch %d proj %d)", c.hidden, c.heads, c.inter, c.image, c.patch, c.proj);
    const size_t item_bytes = static_cast<size_t>(3) * c.image * c.image * 4;
    if (rt.vit_item_bytes != 0 && rt.vit_item_bytes != item_bytes)
        return fail(B200RT_E_UNSUPPORTED, "a second vit model with a different image size is not supported in one runtime");

    auto m = new_model(VIT, c, rt.cap_rows, c.proj);
    m->vcfg = c, m->tokens = T, m->item_bytes = item_bytes;

    // b200rt.weights.vit_blob_layout, plus the patch projection's zero bias
    Layout L;
    L.half(H, PD, &DevWeights::patch_w, &DevWeights::m_patch);
    L.copy(H, &DevWeights::cls);
    L.copy(T * H, &DevWeights::pos);
    L.copy(H, &DevWeights::pre_g);
    L.copy(H, &DevWeights::pre_b);
    for (int l = 0; l < c.layers; ++l) pre_ln_layer(L, l, H, I);
    L.copy(H, &DevWeights::post_g);
    L.copy(H, &DevWeights::post_b);
    L.copy(P * H, &DevWeights::proj_w);
    L.zero(H, &DevWeights::zero_bias);
    if (int rc = load_weights(rt, *m, L, blob, nbytes)) return rc;

    for (size_t g = 0; g < rt.devs.size(); ++g) {
        Dev& d = *rt.devs[g];
        CUDA_TRY(cudaSetDevice(d.id));
        // per-replica image input slots and constants, once
        if (!d.lens_const) {
            std::vector<int32_t> lens(VIT_WAVE_ITEMS, T);
            CUDA_TRY(d.lens_const.alloc(VIT_WAVE_ITEMS * 4));
            CUDA_TRY(cudaMemcpy(d.lens_const, lens.data(), VIT_WAVE_ITEMS * 4, cudaMemcpyHostToDevice));
            if (int rc = make_map_2d(&d.m_im2col, d.ffn, static_cast<uint64_t>(rt.cap_rows) * 4, HIDDEN, 128)) return rc;
        }
        if (!d.copy) CUDA_TRY(d.copy.create());
        for (int sl = 0; sl < NSLOT; ++sl) {
            if (!d.pix_in[sl]) CUDA_TRY(d.pix_in[sl].alloc(VIT_WAVE_ITEMS * m->item_bytes));
            if (!d.ev_pix[sl]) CUDA_TRY(d.ev_pix[sl].create(cudaEventDisableTiming));
        }
    }
    rt.vit_item_bytes = item_bytes;
    return register_model(rt, std::move(m), model_out);
}

int model_load_clip_text(const b200rt_clip_text_config& c, const float* blob, size_t nbytes, int* model_out) {
    Runtime& rt = *g_rt;
    const TextGeometry* tgp = TEXT_GEOMETRIES;
    while (!tgp->causal) ++tgp;  // the one causal geometry of the table
    const TextGeometry& tg = *tgp;
    if (c.hidden != tg.hidden || c.heads != tg.heads || c.inter != tg.inter || c.layers < 1 || c.vocab < 1 || c.proj < 1 || c.proj > 1024)
        return fail(B200RT_E_UNSUPPORTED, "kernels cover the CLIP text tower of clip-vit-base-patch16 / -patch32: hidden=512 heads=8 inter=2048, "
                                          "proj <= 1024 (got hidden %d heads %d inter %d proj %d)", c.hidden, c.heads, c.inter, c.proj);
    if (c.max_pos < 1 || c.max_pos > TEXT_POS_ROWS)
        return fail(B200RT_E_UNSUPPORTED, "max_pos %d outside [1, %d]", c.max_pos, TEXT_POS_ROWS);
    if (c.eos_id < 0 || c.eos_id >= c.vocab) return fail(B200RT_E_INVALID, "eos_id %d outside the vocabulary [0, %d)", c.eos_id, c.vocab);

    auto m = new_model(CLIP_TEXT, c, model_cap_rows(rt.cap_rows, c.hidden), c.proj);
    m->tcfg = c;

    // b200rt.weights.clip_text_blob_layout, with pos padded to TEXT_POS_ROWS zero rows and a zero type row
    const size_t H = c.hidden, I = c.inter;
    Layout L;
    L.copy(c.vocab * H, &DevWeights::word);
    L.copy(c.max_pos * H, &DevWeights::pos);
    L.zero((TEXT_POS_ROWS - c.max_pos) * H);  // the rest of pos: the arena lays it right after pos's max_pos rows
    L.zero(H, &DevWeights::type);
    for (int l = 0; l < c.layers; ++l) pre_ln_layer(L, l, H, I);
    L.copy(H, &DevWeights::post_g);
    L.copy(H, &DevWeights::post_b);
    L.copy(c.proj * H, &DevWeights::proj_w);
    if (int rc = load_weights(rt, *m, L, blob, nbytes)) return rc;
    return register_model(rt, std::move(m), model_out);
}

// Kind "nomic_bert" (HF NomicBertModel): bge-base's geometry, rotary Q / K, SwiGLU MLP, no biases, max_pos <= 8192.
int model_load_nomic(const b200rt_nomic_bert_config& nc, const float* blob, size_t nbytes, bool pool_mean, int* model_out) {
    Runtime& rt = *g_rt;
    const b200rt_bert_config& c = nc.bert;
    if (c.hidden != HIDDEN || c.heads != HEADS || c.inter != 3072 || c.max_pos < 1 || c.max_pos > MAX_SEQ_LONG || c.layers < 1 || c.vocab < 1 ||
        c.type_vocab < 1 || !(nc.rope_theta > 0.f) || !std::isfinite(nc.rope_theta))
        return fail(B200RT_E_UNSUPPORTED,
                    "kernels cover nomic-bert at hidden=768 heads=12 inter=3072, max_pos<=%d, rope_theta > 0 (got hidden %d heads %d inter "
                    "%d max_pos %d rope_theta %g)", MAX_SEQ_LONG, c.hidden, c.heads, c.inter, c.max_pos, static_cast<double>(nc.rope_theta));
    const int S_max = (c.max_pos + 63) / 64 * 64;
    if (rt.cap_rows < S_max)
        return fail(B200RT_E_INVALID, "a nomic_bert model with max_pos %d needs room for one %d-token item, and the workspace holds %d rows: "
                    "initialise with a larger B200RT_INIT_WAVE_ITEMS (now %d)", c.max_pos, S_max, rt.cap_rows, rt.cap_items);

    auto m = new_model(NOMIC_BERT, c, rt.cap_rows, c.hidden);
    m->pool_mean = pool_mean;

    // b200rt.weights.nomic_blob_layout.  QKV of layer l folds the previous layer's ln2 (the embedding LN for l = 0); gate and up
    // (adjacent in the blob) are one [2I, H] entry folding the layer's ln1, interleaved below.  Then the arena-only vectors.
    const size_t H = c.hidden, I = c.inter;
    Layout L;
    L.copy(c.vocab * H, &DevWeights::word);
    L.copy(c.type_vocab * H, &DevWeights::type);
    int ln_g = L.copy(H, &DevWeights::emb_g);
    int ln_b = L.copy(H, &DevWeights::emb_b);
    for (int l = 0; l < c.layers; ++l) {
        const int qkv = L.half(l, 3 * H, H, &LayerW::qkv_w, &LayerW::m_qkv);
        L.fold(qkv, ln_g, ln_b, -1, &LayerW::qkv_c);
        L.half(l, H, H, &LayerW::ao_w, &LayerW::m_ao);
        const int ln1_g = L.copy(l, H, &LayerW::ln1_g), ln1_b = L.copy(l, H, &LayerW::ln1_b);
        const int ff1 = L.half(l, 2 * I, H, &LayerW::ff1_w, &LayerW::m_ff1);
        L.fold(ff1, ln1_g, ln1_b, -1, &LayerW::ff1_c);
        L.half(l, H, I, &LayerW::ff2_w, &LayerW::m_ff2);
        ln_g = L.copy(l, H, &LayerW::ln2_g);
        ln_b = L.copy(l, H, &LayerW::ln2_b);
    }
    L.zero(64 * H, &DevWeights::pos);
    L.zero(H, &DevWeights::zero_bias);
    L.zero(static_cast<size_t>(S_max) * 64, &DevWeights::rope);
    if (int rc = load_weights(rt, *m, L, blob, nbytes)) return rc;

    // The rotary table as HF builds it: inv_freq_i = fp32(1 / fp32(theta^(i/32))), f = fp32(inv_freq_i * pos), then cos / sin of f
    // in double, rounded to fp32.
    std::vector<float2> rope(static_cast<size_t>(S_max) * 32);
    for (int i = 0; i < 32; ++i) {
        const float inv_freq = 1.0f / powf(nc.rope_theta, static_cast<float>(2 * i) / 64.0f);
        for (int p = 0; p < S_max; ++p) {
            const float f = inv_freq * static_cast<float>(p);
            rope[static_cast<size_t>(p) * 32 + i] = make_float2(static_cast<float>(cos(static_cast<double>(f))),
                                                                static_cast<float>(sin(static_cast<double>(f))));
        }
    }
    // gate rows 8k .. 8k+7 -> rows 16k .. 16k+7 and up rows 8k .. 8k+7 -> rows 16k+8 .. 16k+15, and their c alike, through a scratch
    for (size_t g = 0; g < rt.devs.size(); ++g) {
        Dev& d = *rt.devs[g];
        DevWeights& w = m->per_dev[g];
        CUDA_TRY(cudaSetDevice(d.id));
        CUDA_TRY(cudaMemcpyAsync(w.rope, rope.data(), rope.size() * sizeof(float2), cudaMemcpyHostToDevice, d.compute));
        DevMem<__half> sw;  // freed on every return (freeing waits for the device)
        DevMem<float> sc;
        CUDA_TRY(sw.alloc(2 * I * H * 2));
        CUDA_TRY(sc.alloc(2 * I * 4));
        for (int l = 0; l < c.layers; ++l) {
            LayerW& lw = w.layers[l];
            lw.ao_b = lw.ff2_b = w.zero_bias;  // no biases
            for (int part = 0; part < 2; ++part) {  // 0: gate, 1: up
                CUDA_TRY(cudaMemcpy2DAsync(sw + part * 8 * H, 16 * H * 2, lw.ff1_w + part * I * H, 8 * H * 2, 8 * H * 2, I / 8,
                                           cudaMemcpyDeviceToDevice, d.compute));
                CUDA_TRY(cudaMemcpy2DAsync(sc + part * 8, 16 * 4, lw.ff1_c + part * I, 8 * 4, 8 * 4, I / 8, cudaMemcpyDeviceToDevice, d.compute));
            }
            CUDA_TRY(cudaMemcpyAsync(lw.ff1_w, sw, 2 * I * H * 2, cudaMemcpyDeviceToDevice, d.compute));
            CUDA_TRY(cudaMemcpyAsync(lw.ff1_c, sc, 2 * I * 4, cudaMemcpyDeviceToDevice, d.compute));
        }
        CUDA_TRY(cudaStreamSynchronize(d.compute));
    }
    CUDA_TRY(cudaSetDevice(rt.devs[0]->id));
    return register_model(rt, std::move(m), model_out);
}

Runtime* live_rt() {
    if (g_poisoned.load()) {
        fail(B200RT_E_CUDA, "context poisoned by an earlier CUDA error%s%s", g_rt && !g_rt->async_error.empty() ? ": " : "",
             g_rt ? g_rt->async_error.c_str() : "");
        return nullptr;
    }
    if (!g_rt) {
        fail(B200RT_E_STATE, "b200rt_init has not been called");
        return nullptr;
    }
    return g_rt;
}

const Model* get_model(Runtime& rt, int model) {
    std::lock_guard<std::mutex> lk(rt.mu);
    if (model < 0 || model >= static_cast<int>(rt.models.size())) {
        fail(B200RT_E_INVALID, "unknown model handle %d", model);
        return nullptr;
    }
    return rt.models[model].get();
}

// ids [n_items, max_len] with max_len <= S_cap (submit: max_pos; device-resident / debug forwards: max_wave_len) and every
// item's length in [1, min(max_len, max_pos)], its ids inside the vocabulary.
int check_ids(const Model& m, const int32_t* ids, const int32_t* lens, int n_items, int max_len, int S_cap) {
    if (!ids || n_items < 1) return fail(B200RT_E_INVALID, "empty input (n_items=%d)", n_items);
    if (max_len < 1 || max_len > S_cap) return fail(B200RT_E_INVALID, "max_len %d outside [1, %d]", max_len, S_cap);
    const int len_cap = std::min(max_len, m.max_pos);
    for (int i = 0; i < n_items; ++i) {
        const int L = lens ? lens[i] : max_len;
        if (L < 1 || L > len_cap) return fail(B200RT_E_INVALID, "lens[%d] = %d outside [1, %d]", i, L, len_cap);
        const int32_t* row = ids + static_cast<size_t>(i) * max_len;
        for (int j = 0; j < L; ++j)
            if (row[j] < 0 || row[j] >= m.vocab)
                return fail(B200RT_E_INVALID, "ids[%d][%d] = %d outside the vocabulary [0, %d)", i, j, row[j], m.vocab);
    }
    return 0;
}

// Device buffers of one debug entry (b200rt_debug_embed & co.): buffers are filled from the host, zeroed or poisoned in stream
// order on allocation, and freed once the stream has drained when the entry returns, on success or on error.
struct DebugBuffers {
    cudaStream_t stream;
    std::vector<DevMem<void>> ptrs;
    explicit DebugBuffers(cudaStream_t s) : stream(s) {}
    ~DebugBuffers() { cudaStreamSynchronize(stream); }
    template <typename T>
    cudaError_t upload(T** dp, const void* host, size_t bytes, size_t padded = 0) {  // host NULL: zeros; then zeros up to `padded` bytes
        const size_t total = std::max(bytes, padded);
        void* p = nullptr;
        cudaError_t e = alloc(&p, total);
        *dp = static_cast<T*>(p);
        if (e == cudaSuccess && p && (!host || padded > bytes)) e = cudaMemsetAsync(p, 0, total, stream);
        if (e == cudaSuccess && host && bytes) e = cudaMemcpyAsync(p, host, bytes, cudaMemcpyHostToDevice, stream);
        return e;
    }
    template <typename T>
    cudaError_t poisoned(T** dp, size_t bytes) {  // 0xFF bytes, NaN in fp16 and fp32: whatever a kernel leaves unwritten shows
        void* p = nullptr;
        cudaError_t e = alloc(&p, bytes);
        *dp = static_cast<T*>(p);
        return e == cudaSuccess && p ? cudaMemsetAsync(p, 0xFF, bytes, stream) : e;
    }
    cudaError_t download(void* host, const void* dev, size_t bytes) {
        cudaError_t e = cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, stream);
        return e != cudaSuccess ? e : cudaStreamSynchronize(stream);
    }

  private:
    cudaError_t alloc(void** p, size_t bytes) {  // 0 bytes: no buffer, NULL (a launcher judges a NULL operand)
        if (bytes == 0) return cudaSuccess;
        ptrs.emplace_back();
        cudaError_t e = ptrs.back().alloc(bytes);
        if (e == cudaSuccess) *p = ptrs.back();
        return e;
    }
};

// The frame of a debug entry: body(d, b, sms) runs on the live runtime's root replica d, under its lock and with its device
// current, with b a DebugBuffers on d.compute and sms the launch width -- the entry's `sms` (0 = every SM, else 1..SM count;
// an entry without one passes 0).
template <class Body>
int on_root(int sms, Body&& body) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    Dev& d = *rt->devs[0];
    if (sms < 0 || sms > d.sm_count) return fail(B200RT_E_INVALID, "sms must be 0 (every SM) or 1..%d, got %d", d.sm_count, sms);
    std::lock_guard<std::mutex> dl(d.mu);
    CUDA_TRY(cudaSetDevice(d.id));
    DebugBuffers b(d.compute);
    return body(d, b, sms ? sms : d.sm_count);
}

// The mean device time of `iters` (at least one) back-to-back launch() calls on `stream` into *ms_out (may be NULL): one event
// pair around them, synchronised.
template <class Launch>
int time_launches(cudaStream_t stream, int iters, float* ms_out, Launch&& launch) {
    Event e0, e1;
    CUDA_TRY(e0.create());
    CUDA_TRY(e1.create());
    if (iters < 1) iters = 1;
    CUDA_TRY(cudaEventRecord(e0, stream));
    for (int i = 0; i < iters; ++i) LAUNCH_TRY(launch());
    CUDA_TRY(cudaEventRecord(e1, stream));
    CUDA_TRY(cudaEventSynchronize(e1));
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms_out) *ms_out = ms / iters;
    return 0;
}

// Host buffers of a forward trace (b200rt_debug_forward_trace / b200rt_debug_vit_forward_trace, include/b200rt_debug.h).
struct TraceOut {
    uint16_t *yhi, *ylo, *qkv, *ctx, *ffn;
    float *pstats0, *pstats1, *out;
    char* names;
    size_t names_cap;
};

// Runs the first n_launches launches of the forward of host input `in` (ids, lens, segs or pixels) on the root replica d (an
// on_root frame): every workspace buffer and the pooled output are set to 0xFF bytes (NaN in fp16 and fp32) behind the previous
// forward, the launches run on d.compute through forward(), and once the stream has drained, rows = min(M + 256, the model's
// cap_rows) rows of every buffer, at the model's widths (the buffers are used densely at those widths), and the pooled output
// are copied out.
int trace_forward(Dev& d, DebugBuffers& b, const Model& m, const Input& in, int n_launches, const TraceOut& o, int* n_total) {
    const int total = launches_per_forward(m);
    if (n_launches < 0 || n_launches > total) return fail(B200RT_E_INVALID, "n_launches %d outside [0, %d]", n_launches, total);
    if (!o.yhi || !o.ylo || !o.pstats0 || !o.pstats1 || !o.qkv || !o.ctx || !o.ffn || !o.out) return fail(B200RT_E_INVALID, "null output buffer");
    if (n_total) *n_total = total;
    Input din = in;
    if (in.pixels) CUDA_TRY(b.upload(&din.pixels, in.pixels, static_cast<size_t>(in.B) * m.item_bytes));
    else {
        CUDA_TRY(b.upload(&din.ids, in.ids, static_cast<size_t>(in.B) * in.S * 4));
        CUDA_TRY(b.upload(&din.lens, in.lens, static_cast<size_t>(in.B) * 4));
        if (in.segs) CUDA_TRY(b.upload(&din.segs, in.segs, static_cast<size_t>(in.B) * 4));
    }
    const size_t R = g_rt->cap_rows, rows = std::min(static_cast<size_t>(in.B) * in.S + 256, static_cast<size_t>(m.cap_rows));
    const size_t H = m.hidden, I = m.inter, P = H / 128, out_floats = static_cast<size_t>(in.B) * m.out_dim;
    float* dout = nullptr;
    CUDA_TRY(b.poisoned(&dout, out_floats * 4));
    if (d.ev_ws_armed) CUDA_TRY(cudaStreamWaitEvent(d.compute, d.ev_ws, 0));
    for (int i = 0; i < 2; ++i) CUDA_TRY(cudaMemsetAsync(d.pstats[i], 0xFF, R * STAT_PARTS * sizeof(float2), d.compute));
    CUDA_TRY(cudaMemsetAsync(d.yhi, 0xFF, R * HIDDEN * 2, d.compute));
    CUDA_TRY(cudaMemsetAsync(d.ylo, 0xFF, R * HIDDEN * 2, d.compute));
    CUDA_TRY(cudaMemsetAsync(d.qkv, 0xFF, R * QKV_DIM * 2, d.compute));
    CUDA_TRY(cudaMemsetAsync(d.ctx, 0xFF, R * HIDDEN * 2, d.compute));
    CUDA_TRY(cudaMemsetAsync(d.ffn, 0xFF, R * 3072 * 2, d.compute));
    LaunchHook hook;
    hook.stop_after = n_launches;
    uint64_t launches = 0;
    if (int rc = forward(d, m, 0, din, dout, d.compute, launches, &hook)) return rc;
    CUDA_TRY(cudaStreamSynchronize(d.compute));
    CUDA_TRY(cudaMemcpy(o.yhi, d.yhi, rows * H * 2, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(o.ylo, d.ylo, rows * H * 2, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(o.pstats0, d.pstats[0], rows * P * sizeof(float2), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(o.pstats1, d.pstats[1], rows * P * sizeof(float2), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(o.qkv, d.qkv, rows * 3 * H * 2, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(o.ctx, d.ctx, rows * H * 2, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(o.ffn, d.ffn, rows * I * 2, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(o.out, dout, out_floats * 4, cudaMemcpyDeviceToHost));
    if (o.names && o.names_cap) {
        size_t off = 0;
        for (const auto& n : hook.names) {
            if (off + n.size() + 1 > o.names_cap) break;
            memcpy(o.names + off, n.c_str(), n.size() + 1);
            off += n.size() + 1;
        }
        if (off < o.names_cap) o.names[off] = '\0';
    }
    return 0;
}

}  // namespace

// ============================================================================================ C ABI

extern "C" {

int b200rt_init(int n_gpus, uint32_t flags) { return rt_init(nullptr, n_gpus, flags); }
int b200rt_init_devices(const int* devices, int n_gpus, uint32_t flags) { return rt_init(devices, n_gpus, flags); }

int b200rt_num_gpus(void) {
    Runtime* rt = live_rt();
    return rt ? static_cast<int>(rt->devs.size()) : B200RT_E_STATE;
}

int b200rt_wave_capacity_items(void) {
    Runtime* rt = live_rt();
    return rt ? rt->cap_rows / MAX_SEQ : B200RT_E_STATE;
}

int b200rt_model_wave_capacity_items(int model) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    const Model* m = get_model(*rt, model);
    if (!m) return B200RT_E_INVALID;
    return wave_items(*m, MAX_SEQ);
}

int b200rt_model_load(const char* kind, const void* cfg, const void* weights, size_t nbytes, int* model_out) {
    return b200rt_model_load_ex(kind, cfg, weights, nbytes, 0, model_out);
}

int b200rt_model_load_ex(const char* kind, const void* cfg, const void* weights, size_t nbytes, uint32_t flags, int* model_out) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    int k = 0;
    while (k <= CLIP_TEXT && !(kind && strcmp(kind, MODEL_KINDS[k].name) == 0)) ++k;
    if (k > CLIP_TEXT)
        return fail(B200RT_E_UNSUPPORTED, "unknown model kind '%s' (\"bert\", \"bert_classifier\", \"bert_splade\", \"nomic_bert\", \"vit\" or "
                    "\"clip_text\")", kind ? kind : "(null)");
    if (!cfg || !weights || !model_out) return fail(B200RT_E_INVALID, "null argument");
    if (flags & ~B200RT_LOAD_POOL_MEAN) return fail(B200RT_E_INVALID, "unknown load flags 0x%x", flags & ~B200RT_LOAD_POOL_MEAN);
    if (flags && !MODEL_KINDS[k].pool_mean_ok)
        return fail(B200RT_E_INVALID, "load flags 0x%x apply to text encoders of kind \"bert\" or \"nomic_bert\", not \"%s\"", flags,
                    MODEL_KINDS[k].name);
    const bool pool_mean = (flags & B200RT_LOAD_POOL_MEAN) != 0;
    const float* blob = static_cast<const float*>(weights);
    std::lock_guard<std::mutex> dl(rt->devs[0]->mu);  // a load enqueues on the root's compute stream
    switch (static_cast<ModelKind>(k)) {
    case BERT: case BERT_SPLADE: return model_load(static_cast<ModelKind>(k), *static_cast<const b200rt_bert_config*>(cfg), 0, blob, nbytes, pool_mean, model_out);
    case BERT_CLASSIFIER: {
        const auto& cc = *static_cast<const b200rt_bert_classifier_config*>(cfg);
        return model_load(BERT_CLASSIFIER, cc.bert, cc.num_labels, blob, nbytes, false, model_out);
    }
    case NOMIC_BERT: return model_load_nomic(*static_cast<const b200rt_nomic_bert_config*>(cfg), blob, nbytes, pool_mean, model_out);
    case VIT: return model_load_vit(*static_cast<const b200rt_vit_config*>(cfg), blob, nbytes, model_out);
    case CLIP_TEXT: return model_load_clip_text(*static_cast<const b200rt_clip_text_config*>(cfg), blob, nbytes, model_out);
    }
    return fail(B200RT_E_STATE, "internal: no loader for kind \"%s\"", MODEL_KINDS[k].name);
}

// segs [n_items] (b200rt_submit_pairs, classifier models only): item i's second segment starts at token segs[i], 0 <= segs[i] <=
// lens[i]; NULL: one segment.
int check_segs(const Model& m, const int32_t* lens, const int32_t* segs, int n_items, int max_len) {
    if (!segs) return 0;
    if (!takes_segments(m)) return fail(B200RT_E_INVALID, "token segments (segs) apply to classifier models (kind \"bert_classifier\")");
    for (int i = 0; i < n_items; ++i) {
        const int L = lens ? lens[i] : max_len;
        if (segs[i] < 0 || segs[i] > L) return fail(B200RT_E_INVALID, "segs[%d] = %d outside [0, lens[%d] = %d]", i, segs[i], i, L);
    }
    return 0;
}

// A ticket of n_items results of model m, into `out`, for inputs padded to S tokens.
static std::shared_ptr<Ticket> new_ticket(const Model* m, int n_items, int S, float* out) {
    auto t = std::make_shared<Ticket>();
    t->mp = m, t->n_items = n_items, t->S = S, t->out = out;
    t->remaining.store(n_items);
    t->out_pinned = is_pinned(out, static_cast<size_t>(n_items) * m->out_dim * 4);
    return t;
}

// Registers ticket t and queues its runs for the dispatcher.
static int queue_ticket(Runtime& rt, const std::shared_ptr<Ticket>& t, const std::vector<Run>& runs, uint64_t* ticket_out) {
    {
        std::lock_guard<std::mutex> lk(rt.mu);
        if (rt.stopping) return fail(B200RT_E_STATE, "runtime is shutting down");
        t->id = rt.next_ticket++;
        rt.tickets.emplace(t->id, t);
        for (const Run& r : runs) rt.pending.push_back(r);
        rt.last_submit = std::chrono::steady_clock::now();
        *ticket_out = t->id;
    }
    rt.cv_submit.notify_one();
    return 0;
}

static int submit_impl(int model, const int32_t* ids, const int32_t* lens, int n_items, int max_len, float* out,
                       uint32_t flags, uint64_t* ticket_out, const int32_t* segs = nullptr) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    const Model* m = get_model(*rt, model);
    if (!m) return B200RT_E_INVALID;
    if (!out || !ticket_out) return fail(B200RT_E_INVALID, "null out / ticket_out");
    if (m->kind == VIT) return fail(B200RT_E_INVALID, "model %d takes pixels (b200rt_submit_pixels), not token ids", model);
    if (flags & ~static_cast<uint32_t>(B200RT_SUBMIT_BORROW_IDS)) return fail(B200RT_E_INVALID, "unknown submit flags 0x%x", flags);
    if (int rc = check_ids(*m, ids, lens, n_items, max_len, m->max_pos)) return rc;
    if (int rc = check_segs(*m, lens, segs, n_items, max_len)) return rc;
    auto t = new_ticket(m, n_items, max_len, out);
    const size_t id_bytes = static_cast<size_t>(n_items) * max_len * 4;
    if (flags & B200RT_SUBMIT_BORROW_IDS) {  // the caller keeps ids valid and unchanged until the ticket completes
        t->borrowed = true;
        t->ids_ext = ids;
        t->ids_pinned = is_pinned(ids, id_bytes);
    } else {
        t->ids.assign(ids, ids + static_cast<size_t>(n_items) * max_len);
    }
    if (lens) t->lens.assign(lens, lens + n_items);
    else t->lens.assign(n_items, max_len);
    if (segs) t->segs.assign(segs, segs + n_items);
    // runs of items per 64-token length bucket (TEI batches by token budget, un-padded; here every bucket is padded to its
    // own length, so a ragged input wastes at most 63 tokens per item instead of max_len - len)
    std::vector<Run> runs;
    {
        auto bucket_of = [cap = bucket_cap(*m)](int S) { return std::min(cap, (S + 63) / 64 * 64); };
        bool one_bucket = true;
        const int b0 = bucket_of(t->lens[0]);
        for (int i = 1; i < n_items && one_bucket; ++i) one_bucket = bucket_of(t->lens[i]) == b0;
        if (one_bucket) {
            runs.push_back(Run{t, 0, n_items, b0});
        } else {
            t->order.resize(n_items);
            for (int i = 0; i < n_items; ++i) t->order[i] = i;
            std::stable_sort(t->order.begin(), t->order.end(), [&](int a, int b) { return bucket_of(t->lens[a]) < bucket_of(t->lens[b]); });
            for (int i = 0; i < n_items;) {
                const int bk = bucket_of(t->lens[t->order[i]]);
                int j = i;
                while (j < n_items && bucket_of(t->lens[t->order[j]]) == bk) ++j;
                runs.push_back(Run{t, i, j - i, bk});
                i = j;
            }
        }
    }
    return queue_ticket(*rt, t, runs, ticket_out);
}

int b200rt_submit(int model, const int32_t* ids, const int32_t* lens, int n_items, int max_len, float* out,
                  uint64_t* ticket_out) {
    return submit_impl(model, ids, lens, n_items, max_len, out, 0, ticket_out);
}

int b200rt_submit_ex(int model, const int32_t* ids, const int32_t* lens, int n_items, int max_len, float* out,
                     uint32_t flags, uint64_t* ticket_out) {
    return submit_impl(model, ids, lens, n_items, max_len, out, flags, ticket_out);
}

int b200rt_submit_pairs(int model, const int32_t* ids, const int32_t* lens, const int32_t* segs, int n_items, int max_len, float* out,
                        uint32_t flags, uint64_t* ticket_out) {
    return submit_impl(model, ids, lens, n_items, max_len, out, flags, ticket_out, segs);
}

int b200rt_submit_pixels(int model, const float* pixels, int n_items, float* out, uint64_t* ticket_out) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    const Model* m = get_model(*rt, model);
    if (!m) return B200RT_E_INVALID;
    if (m->kind != VIT) return fail(B200RT_E_INVALID, "model %d takes token ids (b200rt_submit), not pixels", model);
    if (!pixels || !out || !ticket_out || n_items < 1) return fail(B200RT_E_INVALID, "null / empty argument");
    auto t = new_ticket(m, n_items, m->tokens, out);
    t->pixels = pixels, t->borrowed = true;
    return queue_ticket(*rt, t, {Run{t, 0, n_items, -m->tokens}}, ticket_out);  // negative bucket keys: image waves never mix with text waves
}

static int reap_locked(Runtime& rt, uint64_t id, const std::shared_ptr<Ticket>& t) {
    for (auto it = rt.finished_unclaimed.begin(); it != rt.finished_unclaimed.end(); ++it)
        if (*it == id) { rt.finished_unclaimed.erase(it); break; }
    rt.tickets.erase(id);
    if (t->status != 0) return fail(t->status, "ticket %llu failed: %s", (unsigned long long)id, t->error.c_str());
    return 0;
}

// Entry/exit bookkeeping of the blocking calls: b200rt_shutdown waits until nobody is inside before it frees the
// runtime (callers are woken with "runtime shut down" first).
struct CallGuard {
    Runtime* rt = nullptr;
    std::unique_lock<std::mutex> lk;
    CallGuard() {
        std::lock_guard<std::mutex> g(g_rt_mu);
        rt = g_rt;
        if (rt) {
            lk = std::unique_lock<std::mutex>(rt->mu);
            rt->active_calls++;
        }
    }
    ~CallGuard() {
        if (rt) {
            if (!lk.owns_lock()) lk.lock();
            rt->active_calls--;
            rt->cv_idle.notify_all();
            lk.unlock();  // the last access to *rt: b200rt_shutdown may free it as soon as the count reaches zero
            lk.release();
        }
    }
};

int b200rt_wait(uint64_t ticket, int timeout_ms) {
    CallGuard g;
    Runtime* rt = g.rt;
    if (!rt) return fail(B200RT_E_STATE, "b200rt_init has not been called");
    auto& lk = g.lk;
    auto it = rt->tickets.find(ticket);
    if (it == rt->tickets.end()) return fail(B200RT_E_INVALID, "unknown or already reaped ticket %llu", (unsigned long long)ticket);
    std::shared_ptr<Ticket> t = it->second;
    // from here on the ticket belongs to this waiter: poll_any will not hand it out
    t->waiters++;
    for (auto f = rt->finished_unclaimed.begin(); f != rt->finished_unclaimed.end(); ++f)
        if (*f == ticket) { rt->finished_unclaimed.erase(f); break; }
    auto pred = [&] { return t->done; };
    bool ok = true;
    if (timeout_ms < 0) rt->cv_done.wait(lk, pred);
    else ok = rt->cv_done.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred);
    t->waiters--;
    if (rt->tickets.find(ticket) == rt->tickets.end())  // a second waiter on the same ticket lost the race
        return fail(B200RT_E_INVALID, "ticket %llu was reaped by another waiter", (unsigned long long)ticket);
    if (!ok) {
        if (t->done && t->waiters == 0) rt->finished_unclaimed.push_back(ticket);  // (cannot happen: done => ok)
        return B200RT_TIMEOUT;
    }
    return reap_locked(*rt, ticket, t);
}

int b200rt_poll_any(uint64_t* ticket_out, int timeout_ms) {
    if (!ticket_out) return fail(B200RT_E_INVALID, "null ticket_out");
    CallGuard g;
    Runtime* rt = g.rt;
    if (!rt) return fail(B200RT_E_STATE, "b200rt_init has not been called");
    auto& lk = g.lk;
    auto pred = [&] { return !rt->finished_unclaimed.empty() || rt->stopping; };
    if (timeout_ms < 0) rt->cv_done.wait(lk, pred);
    else if (!rt->cv_done.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred)) return B200RT_TIMEOUT;
    if (rt->finished_unclaimed.empty()) return fail(B200RT_E_STATE, "runtime shut down");
    const uint64_t id = rt->finished_unclaimed.front();
    auto t = rt->tickets[id];
    *ticket_out = id;
    return reap_locked(*rt, id, t);
}

int b200rt_embed_device(int model, int gpu, const int32_t* d_ids, const int32_t* d_lens, int n_items, int max_len,
                        float* d_out, void* stream) {
    return b200rt_embed_device_pairs(model, gpu, d_ids, d_lens, nullptr, n_items, max_len, d_out, stream);
}

int b200rt_embed_device_pairs(int model, int gpu, const int32_t* d_ids, const int32_t* d_lens, const int32_t* d_segs, int n_items,
                              int max_len, float* d_out, void* stream) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    const Model* m = get_model(*rt, model);
    if (!m) return B200RT_E_INVALID;
    if (gpu < 0 || gpu >= static_cast<int>(rt->devs.size())) return fail(B200RT_E_INVALID, "gpu index %d outside the pool", gpu);
    if (m->kind == VIT) return fail(B200RT_E_UNSUPPORTED, "b200rt_embed_device takes token ids: model %d is not a text encoder", model);
    if (!d_ids || !d_lens || !d_out || n_items < 1 || max_len < 1 || max_len > max_wave_len(*m)) return fail(B200RT_E_INVALID, "bad argument");
    if (d_segs && !takes_segments(*m))
        return fail(B200RT_E_INVALID, "token segments (d_segs) apply to classifier models (kind \"bert_classifier\")");
    Dev& d = *rt->devs[gpu];
    std::lock_guard<std::mutex> dl(d.mu);
    CUDA_TRY(cudaSetDevice(d.id));
    uint64_t launches = 0;
    int rc = forward(d, *m, gpu, Input{d_ids, d_lens, nullptr, n_items, max_len, d_segs}, d_out,
                     stream ? static_cast<cudaStream_t>(stream) : d.compute, launches);
    std::lock_guard<std::mutex> sl(rt->stats_mu);
    rt->stats.kernel_launches += launches;
    return rc;
}

int b200rt_device_sync(int gpu) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    if (gpu < 0 || gpu >= static_cast<int>(rt->devs.size())) return fail(B200RT_E_INVALID, "gpu index %d outside the pool", gpu);
    CUDA_TRY(cudaSetDevice(rt->devs[gpu]->id));
    CUDA_TRY(cudaDeviceSynchronize());
    return 0;
}

void* b200rt_alloc_pinned(size_t nbytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, nbytes) != cudaSuccess) {
        cudaGetLastError();
        fail(B200RT_E_NOMEM, "cudaMallocHost(%zu) failed", nbytes);
        return nullptr;
    }
    {
        std::lock_guard<std::mutex> lk(g_pin_mu);
        g_pinned[reinterpret_cast<uintptr_t>(p)] = nbytes;
    }
    return p;
}
void b200rt_free_pinned(void* p) {
    if (!p) return;
    {
        std::lock_guard<std::mutex> lk(g_pin_mu);
        g_pinned.erase(reinterpret_cast<uintptr_t>(p));
    }
    cudaFreeHost(p);
}

int b200rt_stats(b200rt_stats_t* out) {
    Runtime* rt = g_rt;
    if (!rt) return fail(B200RT_E_STATE, "b200rt_init has not been called");
    if (!out) return fail(B200RT_E_INVALID, "null out");
    std::lock_guard<std::mutex> sl(rt->stats_mu);
    *out = rt->stats;
    return 0;
}

const char* b200rt_last_error(void) { return t_last_error.c_str(); }

void b200rt_shutdown(void) {
    std::lock_guard<std::mutex> glk(g_rt_mu);
    Runtime* rt = g_rt;
    if (!rt) return;
    {
        std::lock_guard<std::mutex> lk(rt->mu);
        rt->stopping = true;
    }
    // 1. no new waves: the dispatcher leaves at its next wait; 2. the completer drains the waves already in flight
    // (their rows still go to live tickets' buffers) and leaves; 3. only then are the remaining tickets failed and
    // their waiters woken, so nothing writes a caller's `out` after that caller was told the runtime is gone.
    rt->cv_submit.notify_all();
    rt->cv_slot.notify_all();
    if (rt->dispatcher.joinable()) rt->dispatcher.join();
    rt->cv_wave.notify_all();
    if (rt->completer.joinable()) rt->completer.join();
    {
        std::unique_lock<std::mutex> lk(rt->mu);
        for (auto& kv : rt->tickets) finish_ticket_locked(*rt, kv.second, B200RT_E_STATE, "runtime shut down");
        rt->pending.clear();
        rt->cv_done.notify_all();
        rt->cv_idle.wait(lk, [&] { return rt->active_calls == 0; });  // blocked b200rt_wait / poll_any callers have left
    }
    for (auto& d : rt->devs) {
        {
            std::lock_guard<std::mutex> ll(d->lmu);
            d->lstop = true;
        }
        d->lcv.notify_all();
        if (d->launcher.joinable()) d->launcher.join();
    }
    for (auto& d : rt->devs) {
        cudaSetDevice(d->id);
        cudaDeviceSynchronize();
    }
    cudaSetDevice(rt->devs[0]->id);  // the caller's thread is left on the root device
    delete rt;  // with every buffer, stream, event and graph of its replicas and models, each released on its own device
    g_rt = nullptr;
}

// ------------------------------------------------------------------------------------------ debug entry points
// Each entry checks what its own host copies need and the debug ABI's policy; the launchers judge every other operand.

int b200rt_debug_gemm(int epi, const uint16_t* a, const uint16_t* w, const float* bias, const float* resid, void* out,
                      int M, int N, int K, int iters, float* ms_out, const float* ln_stats,
                      const float* ln_gamma, const float* ln_beta, float eps, float* stats_out, int sms, int* ctas_out) {
    return b200rt_debug_gemm_ex(epi, a, w, bias, resid, out, M, N, K, iters, ms_out, ln_stats, ln_gamma, ln_beta, eps, stats_out, sms,
                                ctas_out, 0);
}

int b200rt_debug_gemm_ex(int epi, const uint16_t* a, const uint16_t* w, const float* bias, const float* resid, void* out,
                         int M, int N, int K, int iters, float* ms_out, const float* ln_stats,
                         const float* ln_gamma, const float* ln_beta, float eps, float* stats_out, int sms, int* ctas_out, uint32_t flags) {
    return on_root(sms, [&](Dev& d, DebugBuffers& b, int grid_sms) {
        if (flags & ~B200RT_DEBUG_GEMM_LN512) return fail(B200RT_E_INVALID, "unknown gemm flags 0x%x", flags);
        if (!a || !w || !bias || !out || M < 1 || N < 1 || K < 1) return fail(B200RT_E_INVALID, "bad gemm arguments");
        if (epi == 2 && !resid) return fail(B200RT_E_INVALID, "epi 2 needs resid");
        const int ln_w = epi == 2 ? N : K;
        if (ln_stats && ln_w == 512 && !(flags & B200RT_DEBUG_GEMM_LN512))
            return fail(B200RT_E_INVALID, "a 512-wide LayerNorm needs B200RT_DEBUG_GEMM_LN512");
        const size_t Mp = (static_cast<size_t>(M) + 255) / 256 * 256;
        const int parts_in = ln_w / 128, parts_out = N / 128;
        __half *da, *dw, *dhi = nullptr, *dlo = nullptr, *dhi0 = nullptr, *dlo0 = nullptr, *dout = nullptr;
        float *db, *dg = nullptr, *dbt = nullptr;
        float2 *dsi = nullptr, *dso = nullptr;
        CUDA_TRY(b.upload(&da, a, static_cast<size_t>(M) * K * 2, Mp * K * 2));  // rows past M stay zero
        CUDA_TRY(b.upload(&dw, w, static_cast<size_t>(N) * K * 2));
        CUDA_TRY(b.upload(&db, bias, static_cast<size_t>(N) * 4));
        if (ln_stats)  // at least one partial wide, so that a LayerNorm'd width under 128 still reaches the launcher as one
            CUDA_TRY(b.upload(&dsi, ln_stats, static_cast<size_t>(M) * parts_in * sizeof(float2), Mp * std::max(parts_in, 1) * sizeof(float2)));
        if (ln_gamma) CUDA_TRY(b.upload(&dg, ln_gamma, static_cast<size_t>(N) * 4));
        if (ln_beta) CUDA_TRY(b.upload(&dbt, ln_beta, static_cast<size_t>(N) * 4));
        CUtensorMap ta, tb;
        if (int rc = make_map_2d(&ta, da, Mp, K, 128)) return rc;
        if (int rc = make_map_2d(&tb, dw, N, K, 128)) return rc;
        std::vector<__half> hhi, hlo;
        ResEpi res{};  // epi 2: TMA maps over the residual's hi and lo
        OutEpi oe{};   // otherwise: the TMA map the output is stored through, M rows (the poisoned rows past M stay so)
        if (epi == 2) {
            // the residual travels as hi + lo (fp16 + fp16): split on the host, keep a pristine copy for the final launch
            hhi.assign(Mp * N, __float2half_rn(0.f));
            hlo.assign(Mp * N, __float2half_rn(0.f));
            for (size_t i = 0; i < static_cast<size_t>(M) * N; ++i) {
                hhi[i] = __float2half_rn(resid[i]);
                hlo[i] = __float2half_rn(resid[i] - __half2float(hhi[i]));
            }
            CUDA_TRY(b.upload(&dhi0, hhi.data(), Mp * N * 2));
            CUDA_TRY(b.upload(&dlo0, hlo.data(), Mp * N * 2));
            CUDA_TRY(b.upload(&dhi, hhi.data(), Mp * N * 2));
            CUDA_TRY(b.upload(&dlo, hlo.data(), Mp * N * 2));
            CUDA_TRY(b.upload(&dso, nullptr, Mp * parts_out * sizeof(float2)));
            if (int rc = make_map_2d(&res.hi, dhi, Mp, N, 128)) return rc;
            if (int rc = make_map_2d(&res.lo, dlo, Mp, N, 128)) return rc;
        } else {
            CUDA_TRY(b.poisoned(&dout, Mp * N * 2));
            if (int rc = make_map_2d(&oe.out, dout, M, N, 64)) return rc;
        }
        const GemmEpi e{db, dsi, parts_in, dg, dbt, dso, eps};
        auto gemm = [&](int* ctas) {
            return launch_gemm(epi, ta, tb, epi == 2 ? dhi : dout, dlo, epi == 2 ? &res : nullptr, epi == 2 ? nullptr : &oe, e, M, N, K, grid_sms,
                               d.compute, ctas);
        };
        if (int rc = time_launches(d.compute, iters, ms_out, [&] { return gemm(nullptr); })) return rc;  // values drift in place
        if (epi == 2) {  // y = acc + bias + LN(y) in place: reload the residual before the launch whose result is returned
            CUDA_TRY(cudaMemcpyAsync(dhi, dhi0, Mp * N * 2, cudaMemcpyDeviceToDevice, d.compute));
            CUDA_TRY(cudaMemcpyAsync(dlo, dlo0, Mp * N * 2, cudaMemcpyDeviceToDevice, d.compute));
        }
        LAUNCH_TRY(gemm(ctas_out));
        if (epi == 2) {
            CUDA_TRY(b.download(hhi.data(), dhi, Mp * N * 2));
            CUDA_TRY(b.download(hlo.data(), dlo, Mp * N * 2));
            float* o = static_cast<float*>(out);
            for (size_t i = 0; i < static_cast<size_t>(M) * N; ++i) o[i] = __half2float(hhi[i]) + __half2float(hlo[i]);
            if (stats_out) CUDA_TRY(b.download(stats_out, dso, static_cast<size_t>(M) * parts_out * sizeof(float2)));
        } else {
            CUDA_TRY(b.download(out, dout, static_cast<size_t>(M) * N * 2));
        }
        return 0;
    });
}

int b200rt_debug_attention(const uint16_t* qkv, const int32_t* lens, uint16_t* ctx, int B, int S, int iters, float* ms_out, int sms,
                           int head_dim, int heads) {
    return b200rt_debug_attention_ex(qkv, lens, ctx, B, S, iters, ms_out, sms, head_dim, heads, 0);
}

int b200rt_debug_attention_ex(const uint16_t* qkv, const int32_t* lens, uint16_t* ctx, int B, int S, int iters, float* ms_out, int sms,
                              int head_dim, int heads, uint32_t flags) {
    return on_root(sms, [&](Dev& d, DebugBuffers& b, int grid_sms) {
        if (flags & ~B200RT_DEBUG_ATTN_CAUSAL) return fail(B200RT_E_INVALID, "unknown attention flags 0x%x", flags);
        if (head_dim == 0) head_dim = 64;
        if (heads == 0) heads = HEADS;
        if (!qkv || !lens || !ctx || B < 1 || S < 1 || head_dim < 1 || heads < 1) return fail(B200RT_E_INVALID, "bad attention arguments");
        const bool causal = (flags & B200RT_DEBUG_ATTN_CAUSAL) != 0;
        const size_t H = static_cast<size_t>(heads) * head_dim, M = static_cast<size_t>(B) * S;
        __half *dq, *dc;
        int32_t* dl_;
        CUDA_TRY(b.upload(&dq, qkv, M * 3 * H * 2));
        CUDA_TRY(b.poisoned(&dc, M * H * 2));
        CUDA_TRY(b.upload(&dl_, lens, static_cast<size_t>(B) * 4));
        CUtensorMap tq, tc;
        if (int rc = make_map_qkv(&tq, dq, B, S, 3 * H, head_dim)) return rc;
        if (int rc = make_map_qkv(&tc, dc, B, S, H, head_dim)) return rc;
        auto attention = [&] { return launch_attention(tq, tc, dl_, B, S, grid_sms, d.compute, head_dim, heads, causal); };
        LAUNCH_TRY(attention());
        if (int rc = time_launches(d.compute, iters, ms_out, attention)) return rc;
        CUDA_TRY(b.download(ctx, dc, M * H * 2));
        return 0;
    });
}

// embed (segs NULL: type holds one row) and embed_segs (type holds two)
static int debug_embed(const int32_t* ids, const int32_t* segs, const float* word, const float* pos, const float* type, int n_tokens, int S,
                       int vocab, uint16_t* hi_out, uint16_t* lo_out, float* stats_out, int hidden) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!ids || !word || !pos || !type || !hi_out || !lo_out || !stats_out || n_tokens < 1 || S < 1 || vocab < 1 || hidden < 1 ||
            (segs && n_tokens % S))
            return fail(B200RT_E_INVALID, "bad embed arguments (with segs, n_tokens must be a multiple of S)");
        const size_t H = hidden, P = H / 128, rows = static_cast<size_t>(n_tokens);
        int32_t *dids, *dsegs = nullptr;
        float *dw, *dp, *dt;
        __half *dhi, *dlo;
        float2* dst;
        CUDA_TRY(b.upload(&dids, ids, rows * 4));
        if (segs) CUDA_TRY(b.upload(&dsegs, segs, rows / S * 4));  // passed through unchecked: the kernel clamps to [0, S]
        CUDA_TRY(b.upload(&dw, word, static_cast<size_t>(vocab) * H * 4));
        CUDA_TRY(b.upload(&dp, pos, static_cast<size_t>(S) * H * 4));
        CUDA_TRY(b.upload(&dt, type, (segs ? 2 : 1) * H * 4));
        CUDA_TRY(b.upload(&dhi, nullptr, rows * H * 2));
        CUDA_TRY(b.upload(&dlo, nullptr, rows * H * 2));
        CUDA_TRY(b.upload(&dst, nullptr, rows * P * sizeof(float2)));
        LAUNCH_TRY(launch_embed(dids, dw, dp, dt, dhi, dlo, dst, n_tokens, S, vocab, hidden, d.compute, dsegs));
        CUDA_TRY(b.download(hi_out, dhi, rows * H * 2));
        CUDA_TRY(b.download(lo_out, dlo, rows * H * 2));
        CUDA_TRY(b.download(stats_out, dst, rows * P * sizeof(float2)));
        return 0;
    });
}

int b200rt_debug_embed(const int32_t* ids, const float* word, const float* pos, const float* type0, int n_tokens, int S, int vocab,
                       uint16_t* hi_out, uint16_t* lo_out, float* stats_out, int hidden) {
    return debug_embed(ids, nullptr, word, pos, type0, n_tokens, S, vocab, hi_out, lo_out, stats_out, hidden == 0 ? 768 : hidden);
}

int b200rt_debug_embed_segs(const int32_t* ids, const int32_t* segs, const float* word, const float* pos, const float* type, int n_tokens,
                            int S, int vocab, uint16_t* hi_out, uint16_t* lo_out, float* stats_out, int hidden) {
    if (!segs) return fail(B200RT_E_INVALID, "embed_segs needs segs");
    return debug_embed(ids, segs, word, pos, type, n_tokens, S, vocab, hi_out, lo_out, stats_out, hidden);
}

int b200rt_debug_cls_head(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, const float* pool_w,
                          const float* pool_b, const float* cls_w, const float* cls_b, int n_items, int S, int L, float eps, float* out,
                          int hidden, int ctas) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!hi || !lo || !gamma || !beta || !pool_w || !pool_b || !cls_w || !cls_b || !out || n_items < 1 || S < 1 || L < 1 || hidden < 1)
            return fail(B200RT_E_INVALID, "bad cls_head arguments");
        const size_t H = hidden, rows = static_cast<size_t>(n_items) * S;
        __half *dhi, *dlo;
        float *dg, *dbt, *dpw, *dpb, *dcw, *dcb, *dout;
        CUDA_TRY(b.upload(&dhi, hi, rows * H * 2));
        CUDA_TRY(b.upload(&dlo, lo, rows * H * 2));
        CUDA_TRY(b.upload(&dg, gamma, H * 4));
        CUDA_TRY(b.upload(&dbt, beta, H * 4));
        CUDA_TRY(b.upload(&dpw, pool_w, H * H * 4));
        CUDA_TRY(b.upload(&dpb, pool_b, H * 4));
        CUDA_TRY(b.upload(&dcw, cls_w, static_cast<size_t>(L) * H * 4));
        CUDA_TRY(b.upload(&dcb, cls_b, static_cast<size_t>(L) * 4));
        CUDA_TRY(b.poisoned(&dout, static_cast<size_t>(n_items) * L * 4));
        LAUNCH_TRY(launch_cls_head(dhi, dlo, dg, dbt, dpw, dpb, dcw, dcb, dout, n_items, S, L, eps, hidden, d.compute, ctas));
        CUDA_TRY(b.download(out, dout, static_cast<size_t>(n_items) * L * 4));
        return 0;
    });
}

int b200rt_debug_gemm_splade(const uint16_t* a, const uint16_t* w, const float* c, const float* stats, const int32_t* lens, int B, int S,
                             int N, int K, int vocab, float eps, int sms, int iters, float* ms_out, uint32_t* vmax_out, int* ctas_out) {
    return on_root(sms, [&](Dev& d, DebugBuffers& b, int grid_sms) {
        if (!a || !w || !c || !stats || !lens || !vmax_out || B < 1 || S < 1 || N < 1 || K < 1 || vocab < 1)
            return fail(B200RT_E_INVALID, "bad gemm_splade arguments");
        const size_t M = static_cast<size_t>(B) * S, Mp = (M + 255) / 256 * 256, P = K / 128, nmax = static_cast<size_t>(B) * N;
        __half *da, *dw;
        float* dc;
        float2* dst;
        int32_t* dl_;
        uint32_t* dmax;
        CUDA_TRY(b.upload(&da, a, M * K * 2, Mp * K * 2));
        CUDA_TRY(b.upload(&dw, w, static_cast<size_t>(vocab) * K * 2));  // [vocab, K]: the map reads rows past vocab as zeros, as a model's
        CUDA_TRY(b.upload(&dc, c, static_cast<size_t>(N) * 4));
        CUDA_TRY(b.upload(&dst, stats, M * P * sizeof(float2)));
        CUDA_TRY(b.upload(&dl_, lens, static_cast<size_t>(B) * 4));
        CUDA_TRY(b.upload(&dmax, nullptr, nmax * 4));
        CUtensorMap ta, tb;
        if (int rc = make_map_2d(&ta, da, Mp, K, 128)) return rc;
        if (int rc = make_map_2d(&tb, dw, vocab, K, 128)) return rc;
        const GemmEpi e{dc, dst, static_cast<int>(P), nullptr, nullptr, nullptr, eps};
        const SpladeEpi sp{dl_, S, dmax, vocab};
        auto splade = [&](int* ctas) { return launch_gemm_splade(ta, tb, e, sp, static_cast<int>(M), N, K, grid_sms, d.compute, ctas); };
        if (int rc = time_launches(d.compute, iters, ms_out, [&] { return splade(nullptr); })) return rc;
        CUDA_TRY(cudaMemsetAsync(dmax, 0, nmax * 4, d.compute));  // the returned maxima come from one launch on a zeroed buffer
        LAUNCH_TRY(splade(ctas_out));
        CUDA_TRY(b.download(vmax_out, dmax, nmax * 4));
        return 0;
    });
}

// gemm_rope (table non-NULL) and gemm_swiglu: nomic-bert's fused epilogues over a [M, 768] and w [N, 768]
static int debug_nomic_gemm(const uint16_t* a, const uint16_t* w, const float* c, const float* stats, const float* table, int n_pos, int M,
                            int N, int S, int rot_cols, float eps, int sms, uint16_t* out, int* ctas_out) {
    return on_root(sms, [&](Dev& d, DebugBuffers& b, int grid_sms) {
        if (!a || !w || !c || !out || M < 1 || N < 1 || (table && (S < 1 || n_pos < S)))
            return fail(B200RT_E_INVALID, "bad fused GEMM arguments (gemm_rope: n_pos >= S)");
        constexpr size_t K = HIDDEN;
        const size_t Mp = (static_cast<size_t>(M) + 255) / 256 * 256, out_cols = table ? N : N / 2;
        __half *da, *dw, *dout;
        float *dc, *dt = nullptr;
        float2* dst = nullptr;
        CUDA_TRY(b.upload(&da, a, static_cast<size_t>(M) * K * 2, Mp * K * 2));
        CUDA_TRY(b.upload(&dw, w, static_cast<size_t>(N) * K * 2));
        CUDA_TRY(b.upload(&dc, c, static_cast<size_t>(N) * 4));
        if (table) CUDA_TRY(b.upload(&dt, table, static_cast<size_t>(n_pos) * 64 * 4));
        if (stats) CUDA_TRY(b.upload(&dst, stats, static_cast<size_t>(M) * STAT_PARTS * sizeof(float2)));
        CUDA_TRY(b.poisoned(&dout, static_cast<size_t>(M) * out_cols * 2));
        CUtensorMap ta, tb;
        if (int rc = make_map_2d(&ta, da, Mp, K, 128)) return rc;
        if (int rc = make_map_2d(&tb, dw, N, K, 128)) return rc;
        const GemmEpi e{dc, dst, STAT_PARTS, nullptr, nullptr, nullptr, eps};
        LAUNCH_TRY(table ? launch_gemm_rope(ta, tb, dout, e, RopeEpi{reinterpret_cast<const float2*>(dt), S, rot_cols}, M, N, static_cast<int>(K),
                                            grid_sms, d.compute, ctas_out)
                         : launch_gemm_swiglu(ta, tb, dout, e, M, N, static_cast<int>(K), grid_sms, d.compute, ctas_out));
        CUDA_TRY(b.download(out, dout, static_cast<size_t>(M) * out_cols * 2));
        return 0;
    });
}

int b200rt_debug_gemm_rope(const uint16_t* a, const uint16_t* w, const float* c, const float* stats, const float* table, int n_pos, int M,
                           int N, int S, int rot_cols, float eps, int sms, uint16_t* out, int* ctas_out) {
    if (!table) return fail(B200RT_E_INVALID, "gemm_rope needs its table");
    return debug_nomic_gemm(a, w, c, stats, table, n_pos, M, N, S, rot_cols, eps, sms, out, ctas_out);
}

int b200rt_debug_gemm_swiglu(const uint16_t* a, const uint16_t* w, const float* c, const float* stats, int M, int N, float eps, int sms,
                             uint16_t* out, int* ctas_out) {
    return debug_nomic_gemm(a, w, c, stats, nullptr, 0, M, N, 0, 0, eps, sms, out, ctas_out);
}

int b200rt_debug_attention_stream(const uint16_t* qkv, const int32_t* lens, int B, int S, uint16_t* ctx, int sms, int iters, float* ms_out) {
    return on_root(sms, [&](Dev& d, DebugBuffers& b, int grid_sms) {
        if (!qkv || !lens || !ctx || B < 1 || S < 1) return fail(B200RT_E_INVALID, "bad attention_stream arguments");
        const size_t M = static_cast<size_t>(B) * S, H = HIDDEN;
        __half *dq, *dc;
        int32_t* dl_;
        CUDA_TRY(b.upload(&dq, qkv, M * 3 * H * 2));
        CUDA_TRY(b.poisoned(&dc, M * H * 2));
        CUDA_TRY(b.upload(&dl_, lens, static_cast<size_t>(B) * 4));  // passed through unchecked: the kernel clamps to [1, S]
        CUtensorMap tq;
        if (int rc = make_map_qkv(&tq, dq, B, S, 3 * H, 64)) return rc;
        auto attention = [&] { return launch_attention_stream(tq, dc, dl_, B, S, grid_sms, d.compute); };
        LAUNCH_TRY(attention());
        CUDA_TRY(b.download(ctx, dc, M * H * 2));
        return iters > 0 ? time_launches(d.compute, iters, ms_out, attention) : 0;
    });
}

int b200rt_debug_mlm_ln_stats(const uint16_t* u, int n_rows, int hidden, size_t n_max, uint32_t* vmax_out, float* stats_out) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!u || !stats_out || n_rows < 1 || hidden < 1 || (n_max > 0 && !vmax_out)) return fail(B200RT_E_INVALID, "bad mlm_ln_stats arguments");
        const size_t rows = static_cast<size_t>(n_rows), H = hidden, P = H / 128;
        __half* du;
        float2* dst;
        uint32_t* dmax = nullptr;
        CUDA_TRY(b.upload(&du, u, rows * H * 2));
        CUDA_TRY(b.upload(&dst, nullptr, rows * P * sizeof(float2)));
        if (n_max > 0) CUDA_TRY(b.poisoned(&dmax, n_max * 4));
        LAUNCH_TRY(launch_mlm_ln_stats(du, dst, dmax, n_rows, n_max, hidden, d.compute));
        CUDA_TRY(b.download(stats_out, dst, rows * P * sizeof(float2)));
        if (n_max > 0) CUDA_TRY(b.download(vmax_out, dmax, n_max * 4));
        return 0;
    });
}

int b200rt_debug_splade_finalize(const uint32_t* vmax, int n_items, int vpad, int vocab, float* out) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!vmax || !out || n_items < 1 || vocab < 1 || vpad < 1) return fail(B200RT_E_INVALID, "bad splade_finalize arguments");
        const size_t n_out = static_cast<size_t>(n_items) * vocab;
        uint32_t* dmax;
        float* dout;
        CUDA_TRY(b.upload(&dmax, vmax, static_cast<size_t>(n_items) * vpad * 4));
        CUDA_TRY(b.poisoned(&dout, n_out * 4));
        LAUNCH_TRY(launch_splade_finalize(dmax, dout, n_items, vpad, vocab, d.compute));
        CUDA_TRY(b.download(out, dout, n_out * 4));
        return 0;
    });
}

int b200rt_debug_vit_embed(const uint16_t* patch_out, const float* cls, const float* pos, const float* gamma, const float* beta,
                           int n_rows, int T, float eps, uint16_t* hi_out, uint16_t* lo_out, float* stats_out) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!patch_out || !cls || !pos || !gamma || !beta || !hi_out || !lo_out || !stats_out || n_rows < 1 || T < 1)
            return fail(B200RT_E_INVALID, "bad vit_embed arguments");
        const size_t rows = static_cast<size_t>(n_rows);
        __half *dpatch, *dhi, *dlo;
        float *dcls, *dpos, *dg, *dbt;
        float2* dst;
        CUDA_TRY(b.upload(&dpatch, patch_out, rows * HIDDEN * 2));
        CUDA_TRY(b.upload(&dcls, cls, HIDDEN * 4));
        CUDA_TRY(b.upload(&dpos, pos, static_cast<size_t>(T) * HIDDEN * 4));
        CUDA_TRY(b.upload(&dg, gamma, HIDDEN * 4));
        CUDA_TRY(b.upload(&dbt, beta, HIDDEN * 4));
        CUDA_TRY(b.upload(&dhi, nullptr, rows * HIDDEN * 2));
        CUDA_TRY(b.upload(&dlo, nullptr, rows * HIDDEN * 2));
        CUDA_TRY(b.upload(&dst, nullptr, rows * STAT_PARTS * sizeof(float2)));
        LAUNCH_TRY(launch_vit_embed(dpatch, dcls, dpos, dg, dbt, dhi, dlo, dst, n_rows, T, eps, d.compute));
        CUDA_TRY(b.download(hi_out, dhi, rows * HIDDEN * 2));
        CUDA_TRY(b.download(lo_out, dlo, rows * HIDDEN * 2));
        CUDA_TRY(b.download(stats_out, dst, rows * STAT_PARTS * sizeof(float2)));
        return 0;
    });
}

// pool_normalize (lens NULL) and mean_pool_normalize
static int debug_pool(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, const int32_t* lens, int n_items, int S,
                      float eps, float* out, int hidden) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!hi || !lo || !gamma || !beta || !out || n_items < 1 || S < 1 || hidden < 1) return fail(B200RT_E_INVALID, "bad pool arguments");
        const size_t H = hidden, rows = static_cast<size_t>(n_items) * S;
        __half *dhi, *dlo;
        float *dg, *dbt, *dout;
        int32_t* dlens = nullptr;
        CUDA_TRY(b.upload(&dhi, hi, rows * H * 2));
        CUDA_TRY(b.upload(&dlo, lo, rows * H * 2));
        CUDA_TRY(b.upload(&dg, gamma, H * 4));
        CUDA_TRY(b.upload(&dbt, beta, H * 4));
        if (lens) CUDA_TRY(b.upload(&dlens, lens, static_cast<size_t>(n_items) * 4));  // passed through unchecked: the kernel clamps to [1, S]
        CUDA_TRY(b.upload(&dout, nullptr, static_cast<size_t>(n_items) * H * 4));
        LAUNCH_TRY(lens ? launch_mean_pool_normalize(dhi, dlo, dg, dbt, dlens, dout, n_items, S, eps, hidden, d.compute)
                        : launch_pool_normalize(dhi, dlo, dg, dbt, dout, n_items, S, eps, hidden, d.compute));
        CUDA_TRY(b.download(out, dout, static_cast<size_t>(n_items) * H * 4));
        return 0;
    });
}

int b200rt_debug_pool_normalize(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, int n_items, int S,
                                float eps, float* out, int hidden) {
    return debug_pool(hi, lo, gamma, beta, nullptr, n_items, S, eps, out, hidden == 0 ? 768 : hidden);
}

int b200rt_debug_mean_pool_normalize(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, const int32_t* lens,
                                     int n_items, int S, float eps, float* out, int hidden) {
    if (!lens) return fail(B200RT_E_INVALID, "mean_pool_normalize needs lens");
    return debug_pool(hi, lo, gamma, beta, lens, n_items, S, eps, out, hidden == 0 ? 768 : hidden);
}

int b200rt_debug_vit_pool(const uint16_t* hi, const uint16_t* lo, const float* gamma, const float* beta, const float* proj, int n_items,
                          int T, int P, float eps, float* out) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!hi || !lo || !gamma || !beta || !proj || !out || n_items < 1 || T < 1 || P < 1) return fail(B200RT_E_INVALID, "bad vit_pool arguments");
        const size_t rows = static_cast<size_t>(n_items) * T;
        __half *dhi, *dlo;
        float *dg, *dbt, *dproj, *dout;
        CUDA_TRY(b.upload(&dhi, hi, rows * HIDDEN * 2));
        CUDA_TRY(b.upload(&dlo, lo, rows * HIDDEN * 2));
        CUDA_TRY(b.upload(&dg, gamma, HIDDEN * 4));
        CUDA_TRY(b.upload(&dbt, beta, HIDDEN * 4));
        CUDA_TRY(b.upload(&dproj, proj, static_cast<size_t>(P) * HIDDEN * 4));
        CUDA_TRY(b.upload(&dout, nullptr, static_cast<size_t>(n_items) * P * 4));
        LAUNCH_TRY(launch_vit_pool(dhi, dlo, dg, dbt, dproj, dout, n_items, T, P, eps, d.compute));
        CUDA_TRY(b.download(out, dout, static_cast<size_t>(n_items) * P * 4));
        return 0;
    });
}

int b200rt_debug_clip_text_pool(const uint16_t* hi, const uint16_t* lo, const int32_t* ids, const int32_t* lens, const float* gamma,
                                const float* beta, const float* proj, int n_items, int S, int P, float eps, int eos_id, float* out) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!hi || !lo || !ids || !lens || !gamma || !beta || !proj || !out || n_items < 1 || S < 1 || P < 1)
            return fail(B200RT_E_INVALID, "bad clip_text_pool arguments");
        constexpr size_t H = 512;
        const size_t rows = static_cast<size_t>(n_items) * S;
        __half *dhi, *dlo;
        int32_t *dids, *dlens;
        float *dg, *dbt, *dproj, *dout;
        CUDA_TRY(b.upload(&dhi, hi, rows * H * 2));
        CUDA_TRY(b.upload(&dlo, lo, rows * H * 2));
        CUDA_TRY(b.upload(&dids, ids, rows * 4));
        CUDA_TRY(b.upload(&dlens, lens, static_cast<size_t>(n_items) * 4));  // passed through unchecked: the kernel clamps to [1, S]
        CUDA_TRY(b.upload(&dg, gamma, H * 4));
        CUDA_TRY(b.upload(&dbt, beta, H * 4));
        CUDA_TRY(b.upload(&dproj, proj, static_cast<size_t>(P) * H * 4));
        CUDA_TRY(b.upload(&dout, nullptr, static_cast<size_t>(n_items) * P * 4));
        LAUNCH_TRY(launch_clip_text_pool(dhi, dlo, dids, dlens, dg, dbt, dproj, dout, n_items, S, P, eps, eos_id, d.compute));
        CUDA_TRY(b.download(out, dout, static_cast<size_t>(n_items) * P * 4));
        return 0;
    });
}

int b200rt_debug_fold_ln(const float* w, const float* gamma, const float* beta, const float* bias, int N, int K, uint16_t* w_out,
                         float* cvec_out) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        if (!w || !w_out || N < 1 || K < 1) return fail(B200RT_E_INVALID, "bad fold_ln arguments");
        if (gamma && (!beta || !cvec_out)) return fail(B200RT_E_INVALID, "a LayerNorm fold needs beta and cvec_out");
        const size_t n = static_cast<size_t>(N) * K;
        float *dw, *dg = nullptr, *dbt = nullptr, *dbias = nullptr, *dc = nullptr;
        __half* dout;
        CUDA_TRY(b.upload(&dw, w, n * 4));
        if (gamma) {
            CUDA_TRY(b.upload(&dg, gamma, static_cast<size_t>(K) * 4));
            CUDA_TRY(b.upload(&dbt, beta, static_cast<size_t>(K) * 4));
            if (bias) CUDA_TRY(b.upload(&dbias, bias, static_cast<size_t>(N) * 4));
            CUDA_TRY(b.upload(&dc, nullptr, static_cast<size_t>(N) * 4));
        }
        CUDA_TRY(b.upload(&dout, nullptr, n * 2));
        LAUNCH_TRY(launch_fold_ln(dw, dg, dbt, dbias, dout, dc, N, K, d.compute));
        CUDA_TRY(b.download(w_out, dout, n * 2));
        if (gamma) CUDA_TRY(b.download(cvec_out, dc, static_cast<size_t>(N) * 4));
        return 0;
    });
}

int b200rt_debug_forward_trace(int model, const int32_t* ids, const int32_t* lens, int n_items, int max_len, int n_launches,
                               uint16_t* yhi, uint16_t* ylo, float* pstats0, float* pstats1, uint16_t* qkv, uint16_t* ctx,
                               uint16_t* ffn, float* out, char* names_out, size_t names_cap, int* n_total) {
    return b200rt_debug_forward_trace_segs(model, ids, lens, nullptr, n_items, max_len, n_launches, yhi, ylo, pstats0, pstats1, qkv, ctx,
                                           ffn, out, names_out, names_cap, n_total);
}

int b200rt_debug_forward_trace_segs(int model, const int32_t* ids, const int32_t* lens, const int32_t* segs, int n_items, int max_len,
                                    int n_launches, uint16_t* yhi, uint16_t* ylo, float* pstats0, float* pstats1, uint16_t* qkv,
                                    uint16_t* ctx, uint16_t* ffn, float* out, char* names_out, size_t names_cap, int* n_total) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        const Model* m = get_model(*g_rt, model);
        if (!m) return B200RT_E_INVALID;
        if (m->kind == VIT) return fail(B200RT_E_INVALID, "model %d is not a text encoder", model);
        if (int rc = check_ids(*m, ids, lens, n_items, max_len, max_wave_len(*m))) return rc;
        if (int rc = check_segs(*m, lens, segs, n_items, max_len)) return rc;
        if (static_cast<size_t>(n_items) * max_len > static_cast<size_t>(m->cap_rows))
            return fail(B200RT_E_INVALID, "batch exceeds the model's wave capacity");
        std::vector<int32_t> l(n_items, max_len);
        if (lens) l.assign(lens, lens + n_items);
        const TraceOut o{yhi, ylo, qkv, ctx, ffn, pstats0, pstats1, out, names_out, names_cap};
        return trace_forward(d, b, *m, Input{ids, l.data(), nullptr, n_items, max_len, segs}, n_launches, o, n_total);
    });
}

int b200rt_debug_vit_forward_trace(int model, const float* pixels, int n_items, int n_launches, uint16_t* yhi, uint16_t* ylo,
                                   float* pstats0, float* pstats1, uint16_t* qkv, uint16_t* ctx, uint16_t* ffn, float* out,
                                   char* names_out, size_t names_cap, int* n_total) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        const Model* m = get_model(*g_rt, model);
        if (!m) return B200RT_E_INVALID;
        if (m->kind != VIT || !pixels || n_items < 1 || n_items > VIT_WAVE_ITEMS) return fail(B200RT_E_INVALID, "bad arguments");
        const TraceOut o{yhi, ylo, qkv, ctx, ffn, pstats0, pstats1, out, names_out, names_cap};
        return trace_forward(d, b, *m, Input{nullptr, nullptr, pixels, n_items, m->tokens}, n_launches, o, n_total);
    });
}

int b200rt_debug_model_cap_rows(int model) {
    Runtime* rt = live_rt();
    if (!rt) return g_poisoned.load() ? B200RT_E_CUDA : B200RT_E_STATE;
    const Model* m = get_model(*rt, model);
    if (!m) return B200RT_E_INVALID;
    return m->cap_rows;
}

int b200rt_debug_profile_forward(int model, int n_items, int max_len, int iters, char* names_out, size_t names_cap,
                                 float* ms_out, int* n_out, int cap) {
    return on_root(0, [&](Dev& d, DebugBuffers& b, int) {
        const Model* m = get_model(*g_rt, model);
        if (!m) return B200RT_E_INVALID;
        if (m->kind == VIT) return fail(B200RT_E_INVALID, "model %d is not a text encoder", model);
        if (!names_out || !ms_out || !n_out || n_items < 1 || max_len < 1 || max_len > max_wave_len(*m)) return fail(B200RT_E_INVALID, "bad argument");
        const size_t M = static_cast<size_t>(n_items) * max_len;
        if (M > static_cast<size_t>(m->cap_rows)) return fail(B200RT_E_INVALID, "batch exceeds the model's wave capacity");
        std::vector<int32_t> ids(M), l(n_items, std::min(max_len, m->max_pos));  // a clip_text wave may be longer than its items
        uint32_t x = 12345;
        for (auto& v : ids) { x = x * 1664525u + 1013904223u; v = 1000 + static_cast<int32_t>((x >> 8) % (m->vocab - 1000)); }
        int32_t *dids = nullptr, *dlens = nullptr;
        float* dout = nullptr;
        CUDA_TRY(b.upload(&dids, ids.data(), M * 4));
        CUDA_TRY(b.upload(&dlens, l.data(), static_cast<size_t>(n_items) * 4));
        CUDA_TRY(b.upload(&dout, nullptr, static_cast<size_t>(n_items) * m->out_dim * 4));
        if (iters < 1) iters = 1;
        std::map<std::string, double> acc;
        std::vector<std::string> order;
        for (int it = 0; it < iters + 1; ++it) {
            LaunchHook hook;
            hook.timing = true;
            uint64_t launches = 0;
            if (int rc = forward(d, *m, 0, Input{dids, dlens, nullptr, n_items, max_len}, dout, d.compute, launches, &hook)) return rc;
            CUDA_TRY(cudaStreamSynchronize(d.compute));
            for (size_t i = 0; it > 0 && i < hook.names.size(); ++i) {  // the first forward warms up
                float ms = 0;
                cudaEventElapsedTime(&ms, hook.evs[i], hook.evs[i + 1]);
                if (!acc.count(hook.names[i])) order.push_back(hook.names[i]);
                acc[hook.names[i]] += ms;
            }
        }
        size_t off = 0;
        int n = 0;
        for (const auto& name : order) {
            if (n >= cap || off + name.size() + 1 > names_cap) break;
            memcpy(names_out + off, name.c_str(), name.size() + 1);
            off += name.size() + 1;
            ms_out[n++] = static_cast<float>(acc[name] / iters);
        }
        *n_out = n;
        return 0;
    });
}

}  // extern "C"
