"""Which compiled kernel instantiation each launcher selects, restated in Python, and the index of every reachable one.

The launchers in modal-examples_b200/csrc pick a template instantiation from their operands: `launch_gemm` from the epilogue,
N % 256 and the LayerNorm partials it is handed, `launch_attention` from (head_dim, heads, causal), each row launcher from the
row width.  The functions below return what the C++ selects -- a key such as ("gemm_kernel", 0, 256, 6), the kernel's name
and its template arguments in order -- or None where the launcher refuses the operands (cudaErrorInvalidValue).

REACHABLE maps every key some operands can select to the production launches that select it ("bge-small SPLADE transform")
and the debug-entry operands that select it.  tests/test_gpu_instantiations.py checks that this set is exactly the set of
kernels compiled into libb200rt.so, that the rules agree with kernels.h, and runs one conformance test per key."""

GEMM = "gemm_kernel"
ATTN = "attention_kernel"
ATTN_STREAM = "attention_stream_kernel"

EPI_BIAS_F16, EPI_BIAS_GELU_F16, EPI_BIAS_RES_SPLIT, EPI_BIAS_QGELU_F16, EPI_SPLADE_MAX, EPI_ROPE_F16, EPI_SWIGLU_F16 = range(7)


# ------------------------------------------------------------------------------------------------ GEMM

def gemm(epi, N, K, stats_in, parts_in=6):
    """launch_gemm: (GEMM, EPI, BN, PARTS), or None.  `stats_in`: whether e.stats_in is non-NULL (parts_in is
    read only then)."""
    if epi not in (0, 1, 2, 3) or N % 128 or K % 64 or N < 128 or K < 64:
        return None
    ln_width = N if epi == EPI_BIAS_RES_SPLIT else K
    if stats_in and (parts_in not in (8, 6, 4, 3) or parts_in * 128 != ln_width):
        return None
    wide = N % 256 == 0
    if stats_in and parts_in == 8:
        return (GEMM, epi, 256, 8) if epi != EPI_BIAS_QGELU_F16 and wide else None
    if stats_in and parts_in == 4:
        return (GEMM, epi, 256, 4) if epi in (EPI_BIAS_F16, EPI_BIAS_QGELU_F16) and wide else None
    six = not stats_in or parts_in == 6
    return (GEMM, epi, 256 if wide else 128, 6 if six else 3)


def gemm_splade(N, K, stats_in, parts_in=6):
    """launch_gemm_splade: the LayerNorm of A is required, K wide."""
    if N % 256 or K % 64 or not stats_in or parts_in * 128 != K or parts_in not in (6, 3, 8):
        return None
    return (GEMM, EPI_SPLADE_MAX, 256, parts_in)


def gemm_rope(N, K, stats_in, parts_in=6):
    if N % 256 or K != 768 or (stats_in and parts_in != 6):
        return None
    return (GEMM, EPI_ROPE_F16, 256, 6)


def gemm_swiglu(N, K, stats_in, parts_in=6):
    if N % 256 or K != 768 or (stats_in and parts_in != 6):
        return None
    return (GEMM, EPI_SWIGLU_F16, 256, 6)


# ------------------------------------------------------------------------------------------------ attention

ATTN_QT = 128      # query rows per unit when units are split by query tile
ATTN_MAX_S = 512   # launch_attention: S <= MAX_KB * KB
STREAM_MAX_S = 8192


def attention(head_dim, heads, causal):
    """launch_attention: (ATTN, D, NH, CAUSAL), or None."""
    if causal:
        return (ATTN, 64, 8, True) if (head_dim, heads) == (64, 8) else None
    return (ATTN, head_dim, heads, False) if (head_dim, heads) in ((64, 12), (32, 12), (64, 16)) else None


def attention_split(B, S, sms, heads):
    """launch_one: units are split by 128-row query tile when there are fewer (item, head) units than SMs and more than one
    query tile."""
    return B * heads < sms and (S + ATTN_QT - 1) // ATTN_QT > 1


def attention_stream(S):
    return (ATTN_STREAM, 64, 12) if 64 <= S <= STREAM_MAX_S and S % 64 == 0 else None


# ------------------------------------------------------------------------------------------------ row kernels

TEXT_WIDTHS = (768, 384, 1024)


def embed(width, segs):
    ok = width in TEXT_WIDTHS or (width == 512 and not segs)
    return ("embed_kernel", width, bool(segs)) if ok else None


def pool_normalize(width):
    return ("pool_normalize_kernel", width) if width in TEXT_WIDTHS else None


def mean_pool_normalize(width):
    return ("mean_pool_normalize_kernel", width) if width in TEXT_WIDTHS else None


def cls_head(width):
    return ("cls_head_kernel", width) if width in TEXT_WIDTHS else None


def mlm_ln_stats(width):
    return ("mlm_ln_stats_kernel", width) if width in TEXT_WIDTHS else None


def clip_text_pool():
    return ("clip_text_pool_kernel", 512)


def scatter(segs):
    return ("scatter_kernel", bool(segs))


ROW_RULES = {"embed": embed, "pool_normalize": pool_normalize, "mean_pool_normalize": mean_pool_normalize, "cls_head": cls_head,
             "mlm_ln_stats": mlm_ln_stats}

# kernels with a single instantiation: one launcher each, no selection
PLAIN_KERNELS = ("im2col_kernel", "vit_embed_kernel", "vit_pool_kernel", "fold_ln_kernel", "splade_finalize_kernel")


# ------------------------------------------------------------------------------------------------ production launches

# (name, hidden, heads, inter) of the post-LN BERT text geometries; bert, bert_classifier and bert_splade load each of them
BERT_GEOMETRIES = (("bge-base", 768, 12, 3072), ("bge-small", 384, 12, 1536), ("bge-large", 1024, 16, 4096))


def production_launches():
    """Every (model, launch, key) the engine's forward enqueues, from engine.cu's enqueue(): the post-LN text kinds (bert with
    CLS or mean pooling, bert_classifier, bert_splade) at each BERT geometry, nomic-bert, the CLIP text tower and the ViT
    tower.  Post-LN layers fold the previous LayerNorm into QKV / FFN1 and re-apply it in attention-out / FFN2; pre-LN
    layers (CLIP text, ViT) fold LN1 / LN2 and add the residual as is (stats_in NULL)."""
    out = []
    for name, H, NH, I in BERT_GEOMETRIES:
        P = H // 128
        out += [
            (name, "embed", embed(H, False)),
            (f"{name} classifier", "embed of sentence pairs", embed(H, True)),
            (name, "QKV", gemm(EPI_BIAS_F16, 3 * H, H, True, P)),
            (name, "attention", attention(H // NH, NH, False)),
            (name, "attention-out", gemm(EPI_BIAS_RES_SPLIT, H, H, True, P)),
            (name, "FFN1", gemm(EPI_BIAS_GELU_F16, I, H, True, P)),
            (name, "FFN2", gemm(EPI_BIAS_RES_SPLIT, H, I, True, P)),
            (name, "CLS pool", pool_normalize(H)),
            (name, "mean pool", mean_pool_normalize(H)),
            (f"{name} classifier", "pooler / classifier head", cls_head(H)),
            (f"{name} SPLADE", "transform", gemm(EPI_BIAS_GELU_F16, H, H, True, P)),
            (f"{name} SPLADE", "LayerNorm partials of the transform", mlm_ln_stats(H)),
            (f"{name} SPLADE", "decoder vocabulary max", gemm_splade(30720, H, True, P)),
        ]
    out += [
        ("nomic-bert", "embed", embed(768, False)),
        ("nomic-bert", "rotary QKV", gemm_rope(2304, 768, True, 6)),
        ("nomic-bert", "streaming attention", attention_stream(2048)),
        ("nomic-bert", "attention-out", gemm(EPI_BIAS_RES_SPLIT, 768, 768, True, 6)),
        ("nomic-bert", "SwiGLU FFN1", gemm_swiglu(6144, 768, True, 6)),
        ("nomic-bert", "FFN2", gemm(EPI_BIAS_RES_SPLIT, 768, 3072, True, 6)),
        ("nomic-bert", "mean pool", mean_pool_normalize(768)),
        ("nomic-bert", "CLS pool", pool_normalize(768)),
        ("clip-text", "embed", embed(512, False)),
        ("clip-text", "QKV", gemm(EPI_BIAS_F16, 1536, 512, True, 4)),
        ("clip-text", "causal attention", attention(64, 8, True)),
        ("clip-text", "attention-out", gemm(EPI_BIAS_RES_SPLIT, 512, 512, False)),
        ("clip-text", "quick-GELU FFN1", gemm(EPI_BIAS_QGELU_F16, 2048, 512, True, 4)),
        ("clip-text", "FFN2", gemm(EPI_BIAS_RES_SPLIT, 512, 2048, False)),
        ("clip-text", "EOS pool", clip_text_pool()),
        ("vit", "patch GEMM", gemm(EPI_BIAS_F16, 768, 3 * 32 * 32, False)),
        ("vit", "QKV", gemm(EPI_BIAS_F16, 2304, 768, True, 6)),
        ("vit", "attention", attention(64, 12, False)),
        ("vit", "attention-out", gemm(EPI_BIAS_RES_SPLIT, 768, 768, False)),
        ("vit", "quick-GELU FFN1", gemm(EPI_BIAS_QGELU_F16, 3072, 768, True, 6)),
        ("vit", "FFN2", gemm(EPI_BIAS_RES_SPLIT, 768, 3072, False)),
        ("vit", "im2col", ("im2col_kernel",)),
        ("vit", "embed", ("vit_embed_kernel",)),
        ("vit", "pool", ("vit_pool_kernel",)),
        ("every model", "weight load: LayerNorm fold", ("fold_ln_kernel",)),
        ("bert_splade", "log1p of the maxima", ("splade_finalize_kernel",)),
        ("every text model", "wave scatter to the replicas", scatter(False)),
        ("bert_classifier", "wave scatter of sentence pairs", scatter(True)),
    ]
    return out


# ------------------------------------------------------------------------------------------------ debug-entry operands

def _gemm_debug(epi, N, K, ln):
    """b200rt_debug_gemm(_ex) operands: `ln` the LayerNorm partials per row, None for no LayerNorm (ln = 4 needs the
    B200RT_DEBUG_GEMM_LN512 flag)."""
    return dict(entry="debug_gemm", epi=epi, N=N, K=K, ln=ln)


def _gemm_debug_ops():
    """One set of debug operands for each key launch_gemm can select: the LayerNorm'd width (K, or N for epi 2) is ln * 128;
    N = 384 gives the 128-column tile, 768 / 512 / 1024 the 256-column one.  (2, 128, 6) is reachable only without a
    LayerNorm: a 6-partial LayerNorm of the residual makes N = 768, a multiple of 256."""
    ops = {}
    for epi in (0, 1, 2, 3):
        cands = [(768, 768, 6), (384, 384, 3), (384, 768, 6), (768, 384, 3), (512, 512, 4), (1024, 1024, 8), (384, 384, None)]
        for N, K, ln in cands:
            if epi == EPI_BIAS_RES_SPLIT and ln is not None:
                K = N  # the residual LayerNorm is N wide; K is free: take it square
            key = gemm(epi, N, K, ln is not None, ln or 6)
            if key is not None and key not in ops:
                ops[key] = _gemm_debug(epi, N, K, ln)
    return ops


def debug_operands():
    """key -> the debug entry and operands that select it (None for im2col and the wave scatter, which have no debug entry)."""
    ops = _gemm_debug_ops()
    for K, P in ((768, 6), (384, 3), (1024, 8)):
        ops[gemm_splade(512, K, True, P)] = dict(entry="debug_gemm_splade", K=K)
    ops[gemm_rope(2304, 768, True)] = dict(entry="debug_gemm_rope", N=2304)
    ops[gemm_swiglu(6144, 768, True)] = dict(entry="debug_gemm_swiglu", N=6144)
    for d, nh, causal in ((64, 12, False), (32, 12, False), (64, 16, False), (64, 8, True)):
        ops[attention(d, nh, causal)] = dict(entry="debug_attention", head_dim=d, heads=nh, causal=causal)
    ops[attention_stream(512)] = dict(entry="debug_attention_stream")
    for W in TEXT_WIDTHS:
        ops[embed(W, True)] = dict(entry="debug_embed_segs", hidden=W)
        for name in ("pool_normalize", "mean_pool_normalize", "cls_head", "mlm_ln_stats"):
            ops[ROW_RULES[name](W)] = dict(entry=f"debug_{name}", hidden=W)
    for W in TEXT_WIDTHS + (512,):
        ops[embed(W, False)] = dict(entry="debug_embed", hidden=W)
    ops[clip_text_pool()] = dict(entry="debug_clip_text_pool")
    for k in PLAIN_KERNELS:
        ops[(k,)] = dict(entry="debug_" + k[: -len("_kernel")])
    ops[("im2col_kernel",)] = ops[scatter(False)] = ops[scatter(True)] = None
    return ops


def reachable():
    """key -> {"production": ["model: launch", ...], "debug": operands or None}: every instantiation some launch selects."""
    dbg = debug_operands()
    table = {k: {"production": [], "debug": v} for k, v in dbg.items()}
    for model, launch, key in production_launches():
        assert key is not None, (model, launch)
        table.setdefault(key, {"production": [], "debug": None})["production"].append(f"{model}: {launch}")
    return table


REACHABLE = reachable()


def describe(key):
    """gemm_kernel<0, 256, 6> -- the kernel as its C++ name reads."""
    if len(key) == 1:
        return key[0]
    return f"{key[0]}<{', '.join(str(a).lower() for a in key[1:])}>"


def table_lines():
    """The index as text: one line per reachable instantiation."""
    lines = []
    for key in sorted(REACHABLE, key=lambda k: tuple(str(x) for x in k)):
        e = REACHABLE[key]
        prod = "; ".join(e["production"]) or "(debug entry only)"
        dbg = e["debug"]
        dbg = "no debug entry" if dbg is None else ", ".join(f"{k}={v}" for k, v in dbg.items())
        lines.append(f"{describe(key)} | {prod} | {dbg}")
    return lines


if __name__ == "__main__":
    print("\n".join(table_lines()))
    print(f"{len(REACHABLE)} reachable instantiations")
