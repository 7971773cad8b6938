"""GPU parity of the Qwen2-family tokenizer.json path (NFC stage + single-digit Split) through the C ABI: goldens and live `tokenizers`,
NFC segments across the 256-byte windows, threefold growth (cap_tokens, max_tokens_per_request), and the text-in pick of a cl100k, an
r50k and a Qwen2+NFC model in one policy against the tokens-in pick and the oracle."""
import ctypes as C
import json
import os
import random
import unicodedata

import numpy as np
import pytest

from oracle import bpe_ref, orc
from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy, _lib, synth
from smg_b200.policy import TiktokenTokenizer

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
QWEN2 = os.path.join(GOLD, "hf_qwen2_style_tokenizer.json")
VOCAB = os.path.join(GOLD, "synth_vocab.tiktoken")
NFD = lambda s: unicodedata.normalize("NFD", s)   # noqa: E731
MARKS = "̴़्ְּׁ̛̣̰̥֑̀́̂̃̈̊̕͜͡ा"
SPECIALS = ["<|endoftext|>", "<|im_start|>", "<|im_end|>", "<|K|>"]
# decomposed and expanding text (U+1D160, U+FB2C, U+0958), U+212A / U+037E (NFC changes them), jamo, digits and the specials
ALPHABET = list("abcde XYZ 0123456789 '\n\t.,!?-_()") + list(MARKS) + SPECIALS + [NFD(c) for c in "éÅṩệǖ한"] + \
    list("\U0001d160\ufb2c\u0958\u212a\u037e\u1100\u1161\u11a8\uac00\uac01\u00c5\u00e9\uff21\u4f60\U0001f44b\u00b2\u0661")


def _policy(max_tokens_per_request=0, **cfg):
    return CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **cfg), max_tokens_per_request=max_tokens_per_request)


def _live(path=QWEN2):
    ref = pytest.importorskip("tokenizers").Tokenizer.from_file(path)
    return lambda texts: [e.ids for e in ref.encode_batch(texts, add_special_tokens=False)]


def _late_marks():
    """The 108 marks `tokenizers` gives class 0 although Unicode 15 does not: NFC does not move them past a class-1 mark (U+0334)."""
    tk = pytest.importorskip("tokenizers.normalizers").NFC().normalize_str
    marks = [chr(cp) for cp in range(0x300, 0x20000) if unicodedata.combining(chr(cp)) and NFD(chr(cp)) == chr(cp)]
    late = [m for m in marks if (p := "\u4e00" + m + "\u0334" if unicodedata.combining(m) > 1 else "\u4e00\u0301" + m) == tk(p)]
    assert len(late) == 108
    return late


def test_goldens_and_specials_cut_from_the_raw_text():
    """The fixture's goldens.  A mark right after a special is not composed across it; a special that appears only after NFC
    (<|K|> written with U+212A KELVIN SIGN) is ordinary text; a text made only of specials; one digit per piece."""
    tok = _policy().load_hf_tokenizer(QWEN2)
    g = json.load(open(os.path.join(GOLD, "qwen2_vectors.json")))
    for c, ids in zip(g["cases"], tok.encode_batch([c["text"] for c in g["cases"]])):
        assert ids == c["ids"], repr(c["text"][:80])
    sid = {a["content"]: a["id"] for a in json.load(open(QWEN2))["added_tokens"]}
    texts = ["<|im_end|>\u0301", "<|K|>", "<|\u212a|>", "<|im_start|><|im_end|><|K|><|endoftext|>", "", "12345"]
    got = tok.encode_batch(texts)
    assert got[0][0] == sid["<|im_end|>"] and len(got[0]) >= 2 and got[1] == [sid["<|K|>"]] and sid["<|K|>"] not in got[2]
    assert got[3] == [sid[s] for s in ("<|im_start|>", "<|im_end|>", "<|K|>", "<|endoftext|>")] and got[4] == [] and len(got[5]) == 5
    assert got == _live()(texts)


def test_random_texts_and_window_edges_vs_live_tokenizers():
    """900 random texts over an alphabet with the 108 late marks; long mark runs (the long-segment kernel); segments placed across the
    pre-tokenizer's 256-byte windows (which the normalized text shifts) and across the stage's own 256-byte chunks of the raw text."""
    live, tok, rng = _live(), _policy().load_hf_tokenizer(QWEN2), random.Random(2002)
    alphabet = ALPHABET + _late_marks()
    texts = ["".join(rng.choice(alphabet) for _ in range(rng.randint(0, 300))) for _ in range(900)]
    texts += ["x" + "̣́̈" * 1500, "a" + "".join(rng.choice(alphabet[-108:] + list(MARKS)) for _ in range(5000)) + "b",
              "\U0001d160" * 700, NFD("Ångström déjà vu ") * 80, "ᄀ" + "ᅡ" * 600, "1234567890" * 50]
    for k in list(range(248, 264)) + list(range(506, 516)):
        for tail in ("é", NFD("é") + "̣", "\U0001d160" * 3, "a" + "̣́" * 40 + " x", "<|im_end|>́", "क़1",
                     "각", "<|K|>", "<|K|>", " 123 " + "́" * 300):
            texts += ["a" * k + tail, "é" * (k // 2) + tail + "b" * 10, "\U0001d160" * (k // 4) + tail, tail * 30]
    for t, a, b in zip(texts, tok.encode_batch(texts), live(texts)):
        assert a == b, (len(t.encode()), repr(t[-40:]))


def _raw(fn, pol, model, texts, *extra):
    data, offsets = TiktokenTokenizer._ragged(texts)
    return getattr(pol._h.L, fn)(pol._h.p, model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(texts), *extra)


def test_threefold_growth_and_cap_tokens(tmp_path):
    """Without merges every byte of the normalized text is a token: U+1D160 (4 bytes) gives 12.  cap_tokens = 3 × bytes is enough,
    cap_tokens = bytes is the capacity error, and the next call is answered."""
    j = json.load(open(QWEN2))
    j["model"]["merges"] = []
    (tmp_path / "t.json").write_text(json.dumps(j))
    pol = _policy()
    tok = pol.load_hf_tokenizer(str(tmp_path / "t.json"), model="q")
    texts = ["\U0001d160" * k for k in (1, 7, 64, 300)] + ["\ufb2c" * 50, "\u0958" * 90]
    nbytes, want = sum(len(t.encode()) for t in texts), _live(str(tmp_path / "t.json"))(texts)
    for cap, status in ((3 * nbytes, _lib.SUCCESS), (nbytes, _lib.INVALID_ARGUMENT)):
        out, toff = np.zeros(cap, np.uint32), np.zeros(len(texts) + 1, np.uint32)
        assert _raw("smgx_tokenize_batch", pol, b"q", texts, out.ctypes.data_as(C.c_void_p), toff.ctypes.data_as(C.c_void_p), cap, None) == status
        if status == _lib.SUCCESS:
            assert [out[toff[i]:toff[i + 1]].tolist() for i in range(len(texts))] == want and toff[1] == 12 and toff[-1] > nbytes
    assert tok.encode_batch(texts) == want


def _submit(pol, model, texts):
    out, t = np.full(len(texts), -7, np.int32), C.c_uint64()
    data, offsets = TiktokenTokenizer._ragged(texts)
    pol._h.call("smgx_submit_text", model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(texts),
                out.ctypes.data_as(C.c_void_p), None, C.byref(t))
    return out, (data, offsets), t.value


def test_over_length_only_after_normalization():
    """U+0344 (2 bytes) normalizes to U+0308 U+0301: 32 of them are 64 bytes, within max_tokens_per_request = 64, but 96 tokens.  That
    request gets pick -1 and branch 255; the error is reported once — by smgx_select_batch_text itself, or by the smgx_synchronize after
    smgx_submit_text — and the next call on the lane is answered in full."""
    bs, urls = 4, synth.worker_urls(4)
    pol = _policy(64, block_size=bs)
    pol.load_hf_tokenizer(QWEN2, model="q")
    ws = [BasicWorker(u, "q") for u in urls]
    pol.init_workers(ws)
    mon = pol.kv_event_monitor(bs)
    ix = mon.create_indexer("q", 8)
    for u in urls:
        ix.intern_worker(u)
    ix.apply_stored(0, [(1, 12345)])
    pol.set_kv_event_monitor(mon)
    model = pol._push_fleet(ws)
    texts = ["hello world 12", "\u0344" * 32, "naïve café"]
    assert len(texts[1].encode()) == 64 and len(_live()([texts[1]])[0]) > 64 + bs

    def select(ts):
        out, info = np.full(len(ts), -7, np.int32), (_lib.DecisionInfo * len(ts))()
        st = _raw("smgx_select_batch_text", pol, model, ts, out.ctypes.data_as(C.c_void_p), C.cast(info, C.c_void_p), None, None, 0, None)
        return st, out, [info[i].branch for i in range(len(ts))]
    st, out, br = select(texts)
    assert st == _lib.INVALID_ARGUMENT and out[1] == -1 and br[1] == 255 and out[0] >= 0 and out[2] >= 0 and br[0] != 255
    pol._h.call("smgx_synchronize")   # already reported
    st, out, br = select(["short", "text"] * 8)
    assert st == _lib.SUCCESS and (out >= 0).all() and 255 not in br
    out, _keep, ticket = _submit(pol, model, texts)
    pol._h.call("smgx_wait", ticket)
    assert out[1] == -1 and out[0] >= 0 and out[2] >= 0
    assert pol._h.L.smgx_synchronize(pol._h.p, None) == _lib.INVALID_ARGUMENT and pol._h.L.smgx_synchronize(pol._h.p, None) == _lib.SUCCESS
    st, out, _ = select(["after", "the error"] * 8)
    assert st == _lib.SUCCESS and (out >= 0).all()


def test_three_models_text_in_pick_equals_tokens_in_pick_and_oracle():
    """One policy holds "m-cl" (cl100k), "m-r50k" (r50k) and "m-qwen" (the Qwen2+NFC fixture), each with its own KV index.  Per model the
    ids equal its reference (the oracle, or live `tokenizers` for Qwen2) and the text-in pick equals the tokens-in pick and the oracle
    policy's pick; smgx_submit_text calls of the three, interleaved over the stream lanes, pick the same."""
    live, bs, rng = _live(), 4, random.Random(2024)
    cfg = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=bs)
    pol = _policy(**cfg)
    r50k = json.load(open(os.path.join(GOLD, "r50k_vectors.json")))
    urls, models = synth.worker_urls(8), ["m-cl", "m-r50k", "m-qwen"]
    fleets = {m: [BasicWorker(u, m) for u in urls] for m in models}
    pol.init_workers(sum(fleets.values(), []))
    loads = [rng.randint(0, 9) for _ in urls]
    words = "naïve café Ångström 한국어 你好 12345 it's 2024 the quick brown fox x=y+1 \U0001d160 क़ ́".split(" ")
    system = ["<|im_start|>system\n" + " ".join(rng.choice(words) for _ in range(30)) + " 1234567 it'S\n\n<|im_end|>\n" for _ in range(6)]
    texts = [rng.choice(system) + "<|im_start|>user\n" + NFD(" ".join(rng.choice(words) for _ in range(rng.randint(1, 20)))) + "<|im_end|>\n"
             for _ in range(200)] + [" ".join(rng.choice(words) for _ in range(12)) for _ in range(40)]
    mon, picks = pol.kv_event_monitor(bs), {}
    for shift, m in enumerate(models):
        if m == "m-qwen":
            tok, encode = pol.load_hf_tokenizer(QWEN2, model=m), live
        else:
            enc = bpe_ref.CoreBPE(bpe_ref.load_tiktoken_bpe(VOCAB), r50k["specials"], pattern=bpe_ref.CL100K_BASE_PATTERN if m == "m-cl" else r50k["pattern"])
            tok = pol.load_tiktoken_tokenizer(VOCAB, r50k["specials"], model=m, encoding="cl100k_base" if m == "m-cl" else "r50k_base")
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
