"""CPU: the CLIP text tower's host side -- the byte-level BPE tokeniser against HF CLIPTokenizerFast / CLIPTokenizer, the fp64
restatement against HF CLIPTextModelWithProjection and the golden file, both pooling branches, the weight loader and the
infinity_emb adapter's capabilities."""
import hashlib
import importlib.util
import json
import os

import numpy as np
import pytest

import clip_text_refs as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_clip_text_golden", os.path.join(ROOT, "tests", "golden", "make_clip_text_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)

TEXTS = [
    "a photo of a cat", "A PHOTO of a DOG!!", "Hello, world... (really?)", "it's we're they've I'm you'll he'd",
    "numbers 12345 and 3.14159, 1st 2nd", "café naïve résumé Ångström", "東京タワーの写真", "emoji 🐱🐶 party 🎉",
    "tabs\tand\nnewlines   and   runs of   spaces  ", "   leading and trailing   ", "--- ### @@@ $$$ %%% ^^^",
    "mixed 中文 and english words", "a <|endoftext|> b", "<|startoftext|>x<|endoftext|><|endoftext|>", "A <|ENDOFTEXT|> B",
    "x" * 3, " ".join(["word"] * 120), "supercalifragilisticexpialidocious " * 30, "",
]


@pytest.fixture(scope="module")
def vocab_dir(tmp_path_factory):
    """A synthetic CLIP vocabulary: the 512 base symbols, 600 merges learnt from a small corpus, the two special tokens."""
    from infinity_emb.clip_tokenizer import bytes_to_unicode

    bu = bytes_to_unicode()
    syms = list(bu.values())
    vocab = syms + [s + "</w>" for s in syms]
    corpus = " ".join(TEXTS[:6] + ["the quick brown fox jumps over the lazy dog"] * 3 + ["photograph photography photographic"] * 2).lower()
    words = {}
    for w in corpus.split():
        t = tuple("".join(bu[b] for b in w.encode())[:-1]) + ("".join(bu[b] for b in w.encode())[-1] + "</w>",)
        words[t] = words.get(t, 0) + 1
    merges = []
    while len(merges) < 600:
        pairs = {}
        for w, c in words.items():
            for a, b in zip(w, w[1:]):
                pairs[(a, b)] = pairs.get((a, b), 0) + c
        if not pairs:
            break
        best = max(sorted(pairs), key=lambda p: pairs[p])
        merges.append(best)
        vocab.append(best[0] + best[1])
        nw = {}
        for w, c in words.items():
            out, i = [], 0
            while i < len(w):
                if i < len(w) - 1 and (w[i], w[i + 1]) == best:
                    out.append(w[i] + w[i + 1])
                    i += 2
                else:
                    out.append(w[i])
                    i += 1
            nw[tuple(out)] = c
        words = nw
    vocab += ["<|startoftext|>", "<|endoftext|>"]
    d = tmp_path_factory.mktemp("clipvocab")
    json.dump({t: i for i, t in enumerate(vocab)}, open(d / "vocab.json", "w", encoding="utf-8"), ensure_ascii=False)
    with open(d / "merges.txt", "w", encoding="utf-8") as f:
        f.write("#version: 0.2\n" + "\n".join(f"{a} {b}" for a, b in merges) + "\n")
    return str(d)


def _hf(tok, texts):
    enc = tok(texts, padding=True, truncation=True, max_length=77, return_tensors="np")
    return enc["input_ids"].astype(np.int32), enc["attention_mask"].sum(1).astype(np.int32)


def test_tokenizer_matches_clip_tokenizer_fast(vocab_dir):
    from infinity_emb.clip_tokenizer import ClipTokenizer
    from transformers import CLIPTokenizerFast

    ours = ClipTokenizer.from_dir(vocab_dir)
    hf = CLIPTokenizerFast(os.path.join(vocab_dir, "vocab.json"), os.path.join(vocab_dir, "merges.txt"))
    assert not ours.synthetic
    for t in TEXTS:
        ids, lens = ours.batch([t])
        want, wlens = _hf(hf, [t])
        assert lens.tolist() == wlens.tolist() and ids[0, :lens[0]].tolist() == want[0, :wlens[0]].tolist(), t
    ids, lens = ours.batch(TEXTS)
    want, wlens = _hf(hf, TEXTS)
    assert np.array_equal(lens, wlens) and np.array_equal(ids, want)  # padded to the longest with <|endoftext|>, as HF pads
    long = ours.encode(TEXTS[-3])
    assert len(long) == 77 and long[0] == ours.bos_id and long[76] == ours.eos_id  # truncated, end token kept at 76


def test_tokenizer_matches_slow_clip_tokenizer_on_text_both_agree_on(vocab_dir):
    """The slow tokenizer (without ftfy) pre-splits CJK characters and punctuation with BERT's BasicTokenizer; on text where
    that makes no difference it agrees with the fast one, and so with this tokeniser."""
    from infinity_emb.clip_tokenizer import ClipTokenizer
    from transformers import CLIPTokenizer

    ours = ClipTokenizer.from_dir(vocab_dir)
    hf = CLIPTokenizer(os.path.join(vocab_dir, "vocab.json"), os.path.join(vocab_dir, "merges.txt"))
    texts = ["a photo of a cat", "A PHOTO of a DOG", "numbers 12345 and more", "café naïve résumé", "tabs\tand\nnewlines   here",
             " ".join(["word"] * 120)]
    ids, lens = ours.batch(texts)
    want, wlens = _hf(hf, texts)
    assert np.array_equal(lens, wlens) and np.array_equal(ids, want)


def test_tokenizer_offline_fallback_is_clips_base_vocabulary():
    from infinity_emb.clip_tokenizer import ClipTokenizer, bytes_to_unicode

    tok = ClipTokenizer.from_dir(None)
    assert tok.synthetic and tok.bos_id == 49406 and tok.eos_id == 49407
    order = list(bytes_to_unicode())
    ids = tok.encode("Hi, 7")  # "hi" -> h, i</w>; "," -> ,</w>; "7" -> 7</w>
    assert ids == [49406, order.index(ord("h")), 256 + order.index(ord("i")), 256 + order.index(ord(",")), 256 + order.index(ord("7")), 49407]
    assert max(tok.encode("ünïcode 東京 🐱")[1:-1]) < 512


def test_pooling_branches():
    ids = np.array([[49406, 320, 1125, 49407, 49407, 7], [12, 900, 49000, 5, 49000, 49407], [1, 2, 3, 4, 5, 6]], np.int32)
    lens = [6, 5, 1]
    assert T.pooled_positions(ids, lens, 2).tolist() == [3, 2, 0]        # first position of the largest id
    assert T.pooled_positions(ids, lens, 49407).tolist() == [3, 0, 0]    # first end token, 0 when there is none
    assert T.pooled_positions(ids, [2, 5, 1], 49407).tolist() == [0, 0, 0]  # ids past len are never looked at


@pytest.mark.parametrize("case", list(mg.CASES))
def test_oracle_matches_golden_hf_outputs(case):
    golden = np.load(os.path.join(ROOT, "tests", "golden", "clip_text_golden.npz"))
    g, flat, ids, lens = mg.case_inputs(case)
    assert bytes(golden[f"{case}_digest"]) == hashlib.sha256(T.pack_blob(flat, g).tobytes()).digest()
    assert np.array_equal(golden[f"{case}_ids"], ids) and np.array_equal(golden[f"{case}_lens"], lens)
    rel = T.rel_l2(T.forward_np(flat, ids, lens, g), golden[f"{case}_emb"])
    print(f"{case}: numpy fp64 vs HF fp32 rel-L2 {rel.max():.2e}")
    assert rel.max() <= 5e-6, rel


def test_oracle_matches_hf_directly_both_branches():
    g = T.geometry(layers=2, vocab=2000, max_pos=77)
    flat = T.make_weights(g, 5, "trained")
    ids = T.synth_ids([3, 20, 77], 77, seed=4, vocab=2000)
    ids = np.where(ids >= 2000, 1999, ids).astype(np.int32)  # the specials fold into the small vocabulary's last id
    for eos in (2, 1999):
        gg = dict(g, eos_id=eos)
        rel = T.rel_l2(T.forward_np(flat, ids, [3, 20, 77], gg), T.forward_hf(T.build_hf_model(flat, gg), ids, [3, 20, 77]))
        assert rel.max() <= 5e-6, (eos, rel)


def test_weight_loader_takes_clip_model_and_text_model_with_projection_keys():
    from b200rt import weights as W

    from oracle import clip_ref as C

    g = T.geometry(layers=2, vocab=600, max_pos=77)
    flat = T.make_weights(g, 1, "trained")
    want = T.pack_blob(flat, g)
    hf = T.build_hf_model(flat, g)  # CLIPTextModelWithProjection's own state dict
    g1, b1 = W.load_clip_text_state_dict({k: v for k, v in hf.state_dict().items()}, eps=g["eps"], eos_id=2)
    assert np.array_equal(b1, want) and {k: g1[k] for k in g} == g
    vg = C.VitGeometry(layers=1)
    sd = dict(C.flat_to_hf_state(C.make_weights(vg, 0), vg), **T.flat_to_hf_state(flat, g), logit_scale=np.array(4.6, np.float32))
    g2, b2 = W.load_clip_text_state_dict(sd)  # a CLIPModel's: both towers and logit_scale
    assert np.array_equal(b2, want) and g2["layers"] == 2 and g2["heads"] == 8 and g2["proj"] == 512
    sd.pop("text_projection.weight")
    with pytest.raises(KeyError):
        W.load_clip_text_state_dict(sd)


def test_eos_id_comes_from_the_snapshot_config(tmp_path):
    from b200rt import weights as W

    assert W.clip_text_config_from_dir(str(tmp_path))["eos_id"] == 2
    json.dump({"text_config": {"eos_token_id": 49407, "layer_norm_eps": 1e-5, "num_attention_heads": 8}}, open(tmp_path / "config.json", "w"))
    assert W.clip_text_config_from_dir(str(tmp_path)) == dict(eps=1e-5, heads=8, eos_id=49407)


def test_blob_layout_sizes():
    from b200rt import weights as W

    g = W.CLIP_TEXT_B16_GEOMETRY
    n = W.clip_text_blob_numel(g)
    assert n == 49408 * 512 + 77 * 512 + 12 * (4 * 512 * 512 + 2 * 512 * 2048 + 9 * 512 + 2048) + 2 * 512 + 512 * 512
    small = dict(g, vocab=1000, layers=2)
    for seed in (0, 7):
        assert np.array_equal(W.random_clip_text_blob(small, seed), T.pack_blob(T.make_weights(small, seed, "hf"), small))


def test_flops_per_item_at_bucket_128():
    """The shape-derived work figure quoted in DESIGN.md and tools/clip_text_bench.py: 10.07 GFLOP per 128-token item."""
    S, H, I, L = 128, 512, 2048, 12
    per_layer = 2 * S * (3 * H * H + H * H + 2 * H * I) + 2 * 2 * S * S * H
    assert abs(L * per_layer / 1e9 - 10.07) < 0.005


def test_infinity_engine_advertises_text_and_image_embedding():
    from infinity_emb import AsyncEmbeddingEngine, EngineArgs

    assert AsyncEmbeddingEngine.from_args(EngineArgs()).capabilities == {"embed", "image_embed"}
