"""GPU parity of the SentencePiece-style tokenizer.json path (Llama 2, Mistral, TinyLlama: ▁ normalization, cut at ▁, character-level
symbols with byte fallback) through the C ABI: goldens and live `tokenizers` for the legacy shape and the Metaspace variants, every merge
tier, the twofold token bound (cap_tokens, max_tokens_per_request), untouched output past the written tokens, and the text-in pick of a
Llama-2-style, a cl100k and a Qwen2+NFC model in one policy against the tokens-in pick and the oracle.  An optional test loads a real file
named by $SMGX_REAL_SP_TOKENIZER_JSON."""
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

from oracle import bpe_ref, orc
from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy, _lib, synth
from smg_b200.policy import TiktokenTokenizer

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
LLAMA2 = os.path.join(GOLD, "hf_llama2_style_tokenizer.json")
QWEN2 = os.path.join(GOLD, "hf_qwen2_style_tokenizer.json")
VOCAB = os.path.join(GOLD, "synth_vocab.tiktoken")
SPECIALS = ["<unk>", "<s>", "</s>", "<|user|>", "<|assistant|>"]
ALPHABET = [" ", " ", " ", "  ", "▁", "\t", "\n", "\r\n", "the", "quick", "brown", "fox", "a", "e", "é", "é", "café", "中文", "你好", "龍",
            "😀", "👋🌍", "<0x41>", "x=y+1", "12345", "    "] + SPECIALS
VARIANTS = ["legacy", "metaspace-first-nosplit", "metaspace-always-nosplit", "metaspace-first-split"]


def _variant(name, tmp_path, merges=True):
    j = json.load(open(LLAMA2))
    if name != "legacy":
        _, scheme, split = name.split("-")
        j["normalizer"] = None
        j["pre_tokenizer"] = {"type": "Metaspace", "replacement": "▁", "prepend_scheme": scheme, "split": split == "split"}
    if not merges:
        j["model"]["merges"] = []
    p = tmp_path / f"{name}{'' if merges else '-nomerges'}.json"
    p.write_text(json.dumps(j))
    return str(p)


def _policy(max_tokens_per_request=0, **cfg):
    return CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **cfg), max_tokens_per_request=max_tokens_per_request)


def _live(path):
    ref = pytest.importorskip("tokenizers").Tokenizer.from_file(path)
    return lambda texts: [e.ids for e in ref.encode_batch(texts, add_special_tokens=False)]


def _raw(fn, pol, model, texts, *extra):
    data, offsets = TiktokenTokenizer._ragged(texts)
    return getattr(pol._h.L, fn)(pol._h.p, model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(texts), *extra)


@pytest.mark.parametrize("name", VARIANTS)
def test_goldens(name, tmp_path):
    g = json.load(open(os.path.join(GOLD, "llama2_vectors.json")))
    tok = _policy().load_hf_tokenizer(_variant(name, tmp_path))
    for c, got, want in zip(g["cases"], tok.encode_batch([c["text"] for c in g["cases"]]), g["variants"][name]):
        assert got == want, repr(c["text"][:80])


@pytest.mark.parametrize("name", VARIANTS)
def test_random_texts_and_every_tier_vs_live_tokenizers(name, tmp_path):
    """500 random texts; pieces of every tier by symbol count (≤15 per thread, ≤32 per warp, ≤256 in shared memory, beyond that in global
    memory): space-free runs of vocabulary and byte-fallback characters, all-space stretches, placed across the 256-byte windows."""
    path = _variant(name, tmp_path)
    live, tok, rng = _live(path), _policy().load_hf_tokenizer(path), random.Random(VARIANTS.index(name))
    texts = ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, 120))) for _ in range(500)]
    for k in (1, 2, 14, 15, 16, 31, 32, 33, 100, 255, 256, 257, 700):
        texts += ["x" * k, " y" + "龍" * k, "中" * k + " z", "😀" * k, " " * k, "<s>" + " " * k + "</s>", "a" + "é" * k, "▁" * k]
    for k in list(range(250, 262)) + [510, 511, 512, 1030]:   # normalized text shifts pieces across windows and raw chunks
        texts += ["a" * k + " b c", " " * k + "中文 x", "<s>" * (k // 3) + " hi", "é" * (k // 2) + " 😀 x"]
    for t, a, b in zip(texts, tok.encode_batch(texts), live(texts)):
        assert a == b, (name, len(t.encode()), repr(t[:60]))


def test_twofold_token_bound_and_cap_tokens(tmp_path):
    """Without merges a space between specials gives "▁▁" — two tokens from one byte (legacy shape) — and a byte-fallback character its
    bytes plus the prepended ▁.  cap_tokens = 2 × bytes is enough and is reached exactly; one less is the capacity error, after which
    the next call is answered.  Poisoned output past the written tokens stays untouched."""
    path = _variant("legacy", tmp_path, merges=False)
    pol = _policy()
    tok = pol.load_hf_tokenizer(path, model="l")
    between = ["<s> </s> <s>", "<|user|> <|assistant|> ", " <s> ", " " * 7, "<s>" + " " * 300 + "</s>"]
    assert tok.encode_batch(between) == _live(path)(between)
    texts = [" "] * 64   # every request one space: the bound is reached exactly
    nbytes, want = 64, _live(path)(texts)
    assert sum(len(w) for w in want) == 2 * nbytes
    for cap, status in ((2 * nbytes + 16, _lib.SUCCESS), (2 * nbytes, _lib.SUCCESS), (2 * nbytes - 1, _lib.INVALID_ARGUMENT)):
        out, toff = np.full(cap + 16, 0xDEADBEEF, np.uint32), np.zeros(len(texts) + 1, np.uint32)
        assert _raw("smgx_tokenize_batch", pol, b"l", texts, out.ctypes.data_as(C.c_void_p), toff.ctypes.data_as(C.c_void_p), cap, None) == status
        if status == _lib.SUCCESS:
            assert [out[toff[i]:toff[i + 1]].tolist() for i in range(len(texts))] == want and toff[-1] == 2 * nbytes
            assert (out[2 * nbytes:] == 0xDEADBEEF).all()
    assert tok.encode_batch(texts) == want
    mixed = ["😀", "<s>😀</s>", "\t\t", " 龍 "]
    assert tok.encode_batch(mixed) == _live(path)(mixed)


def _submit(pol, model, texts):
    out, t = np.full(len(texts), -7, np.int32), C.c_uint64()
    data, offsets = TiktokenTokenizer._ragged(texts)
    pol._h.call("smgx_submit_text", model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(texts),
                out.ctypes.data_as(C.c_void_p), None, C.byref(t))
    return out, (data, offsets), t.value


def test_over_length_only_after_normalization():
    """16 emoji are 64 bytes, within max_tokens_per_request = 64, but 65 tokens (the prepended ▁ and 64 byte-fallback tokens) — with
    one-token blocks, 65 blocks where the hash row holds 64.  (A stretch of L bytes has at most L + 1 tokens, so only the block size 1 lets
    the one extra token cross a block boundary.)  That request gets pick -1 and branch 255; the error is reported once — by
    smgx_select_batch_text itself, or by the smgx_synchronize after smgx_submit_text — and the next call is answered in full."""
    bs, urls = 1, synth.worker_urls(4)
    pol = _policy(64, block_size=bs)
    pol.load_hf_tokenizer(LLAMA2, model="l")
    ws = [BasicWorker(u, "l") for u in urls]
    pol.init_workers(ws)
    mon = pol.kv_event_monitor(bs)
    ix = mon.create_indexer("l", 8)
    for u in urls:
        ix.intern_worker(u)
    ix.apply_stored(0, [(1, 12345)])
    pol.set_kv_event_monitor(mon)
    model = pol._push_fleet(ws)
    texts = ["hello world", "😀" * 16, "café 中文"]
    assert len(texts[1].encode()) == 64 and len(_live(LLAMA2)([texts[1]])[0]) == 65

    def select(ts):
        out, info = np.full(len(ts), -7, np.int32), (_lib.DecisionInfo * len(ts))()
        st = _raw("smgx_select_batch_text", pol, model, ts, out.ctypes.data_as(C.c_void_p), C.cast(info, C.c_void_p), None, None, 0, None)
        return st, out, [info[i].branch for i in range(len(ts))]
    st, out, br = select(texts)
    assert st == _lib.INVALID_ARGUMENT and out[1] == -1 and br[1] == 255 and out[0] >= 0 and out[2] >= 0 and br[0] != 255
    pol._h.call("smgx_synchronize")
    st, out, br = select(["short", "text"] * 8)
    assert st == _lib.SUCCESS and (out >= 0).all() and 255 not in br
    out, _keep, ticket = _submit(pol, model, texts)
    pol._h.call("smgx_wait", ticket)
    assert out[1] == -1 and out[0] >= 0 and out[2] >= 0
    assert pol._h.L.smgx_synchronize(pol._h.p, None) == _lib.INVALID_ARGUMENT and pol._h.L.smgx_synchronize(pol._h.p, None) == _lib.SUCCESS


def test_three_models_text_in_pick_equals_tokens_in_pick_and_oracle():
    """One policy holds "m-llama" (the Llama-2-style fixture), "m-cl" (cl100k) and "m-qwen" (Qwen2+NFC), each with its own KV index.  Per
    model the ids equal its reference and the text-in pick equals the tokens-in pick and the oracle policy's pick; smgx_submit_text calls
    of the three, interleaved over the stream lanes, pick the same."""
    bs, rng = 4, random.Random(2025)
    cfg = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=bs)
    pol = _policy(**cfg)
    r50k = json.load(open(os.path.join(GOLD, "r50k_vectors.json")))
    urls, models = synth.worker_urls(8), ["m-llama", "m-cl", "m-qwen"]
    fleets = {m: [BasicWorker(u, m) for u in urls] for m in models}
    pol.init_workers(sum(fleets.values(), []))
    loads = [rng.randint(0, 9) for _ in urls]
    words = "the quick brown fox naïve café 中文 你好 龍 12345 it's x=y+1 😀 👋 \t".split(" ") + ["", "  "]
    system = ["<s><|user|>\n" + " ".join(rng.choice(words) for _ in range(30)) + "</s>\n" for _ in range(6)]
    texts = [rng.choice(system) + "<|assistant|>\n" + " ".join(rng.choice(words) for _ in range(rng.randint(1, 20))) + "</s>"
             for _ in range(200)] + [" ".join(rng.choice(words) for _ in range(12)) for _ in range(40)]
    mon, picks = pol.kv_event_monitor(bs), {}
    for shift, m in enumerate(models):
        if m == "m-llama":
            tok, encode = pol.load_hf_tokenizer(LLAMA2, model=m), _live(LLAMA2)
        elif m == "m-qwen":
            tok, encode = pol.load_hf_tokenizer(QWEN2, model=m), _live(QWEN2)
        else:
            enc = bpe_ref.CoreBPE(bpe_ref.load_tiktoken_bpe(VOCAB), r50k["specials"], pattern=bpe_ref.CL100K_BASE_PATTERN)
            tok = pol.load_tiktoken_tokenizer(VOCAB, r50k["specials"], model=m, encoding="cl100k_base")
            encode = lambda ts, enc=enc: [enc.encode_with_special_tokens(t) for t in ts]   # noqa: E731
        ix, op, oix = mon.create_indexer(m, 8), orc.CacheAwarePolicy(eviction_interval_secs=0, **cfg), orc.PositionalIndexer(8)
        op.set_workers(urls, models=[m] * 8)
        op.attach_indexer(m, oix)
        op.set_kv_event_monitor(True)
        for u in urls:
            assert ix.intern_worker(u) == oix.intern_worker(u)
        seq = 1
        for k, ids in enumerate(encode(system)):   # the models cache the prompts on different workers
            hs = orc.compute_request_content_hashes(ids, bs)
            blocks = [(seq + i, hs[i]) for i in range(len(ids) // bs)]
            seq += len(blocks)
            for w in ((k + 3 * shift) % 8, (k + 3 * shift + 5) % 8):
                ix.apply_stored(w, blocks)
                oix.apply_stored(w, blocks)
        for w, l in zip(fleets[m], loads):
            w.set_load(l)
        op.set_state(loads, [1] * 8, [1] * 8)
        pol.set_kv_event_monitor(mon)
        idx_text, _, toks = pol.select_worker_batch_text(fleets[m], texts)
        assert toks == encode(texts) == tok.encode_batch(texts), m
        idx_tok, _ = pol.select_worker_batch(fleets[m], toks)
        offs = np.zeros(len(toks) + 1, np.uint64)
        np.cumsum([len(t) for t in toks], out=offs[1:])
        want, br, _, _ = op.select_batch_tokens(np.concatenate([np.asarray(t, np.uint32) for t in toks]), offs)
        assert np.array_equal(idx_text, idx_tok) and np.array_equal(idx_text, want) and (np.asarray(br) == 2).sum() > 100, m
        picks[m] = idx_text
    depth, subs = pol._h.L.smgx_pipeline_depth(pol._h.p), []
    for i, m in enumerate(models * 3):   # as many in flight as there are lanes
        if len(subs) >= depth:
            pol._h.call("smgx_wait", subs[-depth][2])
        subs.append(_submit(pol, pol._push_fleet(fleets[m]), texts[i // 3::3]) + (m, i // 3))
    for s in subs[-depth:]:
        pol._h.call("smgx_wait", s[2])
    for out, _keep, _t, m, k in subs:
        assert np.array_equal(out, picks[m][k::3]), (m, k)


@pytest.mark.skipif(not os.environ.get("SMGX_REAL_SP_TOKENIZER_JSON"), reason="set SMGX_REAL_SP_TOKENIZER_JSON to a real Llama-2 / Mistral / "
                    "TinyLlama tokenizer.json")
def test_real_sentencepiece_tokenizer_json():
    """A real file either loads — its merges pass the exactness check — and then matches live `tokenizers`, or is refused loudly."""
    path = os.environ["SMGX_REAL_SP_TOKENIZER_JSON"]
    try:
        tok = _policy().load_hf_tokenizer(path)
    except ValueError as e:
        pytest.fail(f"refused: {e}")
    rng = random.Random(5)
    texts = ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, 200))) for _ in range(400)]
    texts += ["Hello world! How are you today?", "  def main():\n\treturn 0", "日本語のテキスト", "🧑‍💻 ünïcödé ≠ ∑"]
    assert tok.encode_batch(texts) == _live(path)(texts)
