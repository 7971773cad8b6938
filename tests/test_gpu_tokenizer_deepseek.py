"""GPU parity of the DeepSeek-V3-family tokenizer.json path (the chain of three Splits: digit triples, kana/CJK runs, words) through the C
ABI: goldens and live `tokenizers`, digit / kana / letter / whitespace runs across the pre-tokenizer's 256-byte windows, specials inside
digit triples, both ignore_merges values, cap_tokens = total bytes, and the text-in pick of a cl100k, a Qwen2+NFC and a DeepSeek model in
one policy against the tokens-in pick and the oracle.  An optional test loads a real file named by $SMGX_REAL_DEEPSEEK_TOKENIZER_JSON."""
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
DEEPSEEK = os.path.join(GOLD, "hf_deepseek_v3_style_tokenizer.json")
QWEN2 = os.path.join(GOLD, "hf_qwen2_style_tokenizer.json")
VOCAB = os.path.join(GOLD, "synth_vocab.tiktoken")
BOS, EOS, USER, ASSISTANT = "<｜begin▁of▁sentence｜>", "<｜end▁of▁sentence｜>", "<｜User｜>", "<｜Assistant｜>"
# digits of several scripts, kana/CJK with the punctuation, symbols, marks and unassigned code points inside the ranges, ASCII punctuation,
# letters, marks, format and control characters, whitespace of every kind, and the specials
ALPHABET = list("abcXYZ é0123456789١٢٣²³½Ⅳ０中文テスト・゠゛ゞ゚゗鿿가.,!?'\"-_()<|>$+^`~@#\\/{}「」、。́̀ि\x00\x01​‍﻿  \n\n\r\t\x0b\x85\xa0　") + \
    ["\U0001f44b", "\U000e0001", BOS, EOS, USER, ASSISTANT]


def _policy(**cfg):
    return CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **cfg))


def _live(path=DEEPSEEK):
    ref = pytest.importorskip("tokenizers").Tokenizer.from_file(path)
    return lambda texts: [e.ids for e in ref.encode_batch(texts, add_special_tokens=False)]


def _raw(fn, pol, model, texts, *extra):
    data, offsets = TiktokenTokenizer._ragged(texts)
    return getattr(pol._h.L, fn)(pol._h.p, model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(texts), *extra)


def test_goldens_and_specials_inside_digit_and_cjk_runs():
    """The fixture's goldens; a special cuts a digit run, and the triples restart after it; specials alone; the empty text."""
    tok = _policy().load_hf_tokenizer(DEEPSEEK)
    g = json.load(open(os.path.join(GOLD, "deepseek_vectors.json")))
    for c, ids in zip(g["cases"], tok.encode_batch([c["text"] for c in g["cases"]])):
        assert ids == c["ids"], repr(c["text"][:80])
    sid = {a["content"]: a["id"] for a in json.load(open(DEEPSEEK))["added_tokens"]}
    texts = ["1234" + BOS + "56789", "12" + EOS + "3" + EOS + "4567", "中文" + USER + "テスト・" + ASSISTANT + "ア", BOS + EOS + USER + ASSISTANT,
             "", "9" * 7 + BOS]
    got = tok.encode_batch(texts)
    assert sid[BOS] in got[0] and got[3] == [sid[s] for s in (BOS, EOS, USER, ASSISTANT)] and got[4] == [] and got[5][-1] == sid[BOS]
    assert got == _live()(texts)


def test_random_texts_and_runs_across_windows_vs_live_tokenizers():
    """700 random texts; digit, kana/CJK, letter and whitespace runs placed across the 256-byte windows of the pre-tokenizer, and single
    digit runs longer than a window."""
    live, tok, rng = _live(), _policy().load_hf_tokenizer(DEEPSEEK), random.Random(2025)
    texts = ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, 300))) for _ in range(700)]
    texts += ["1" * 700, "x" + "1234567890" * 90, "١" * 400, "中" * 300 + "テスト・" * 60, " " * 700 + "a", "\n" * 600 + "  x"]
    for k in list(range(246, 266)) + list(range(505, 515)):
        for run in ("1234567", "١٢٣٤٥", "中文テスト・ア", "abcdefé́", "   \n\n  ", "  ", ".,!?abc", "x\x00\x01 .", "12" + BOS + "345"):
            texts += ["a" * k + run + "b", "1" * k + run, "é" * (k // 2) + run + " 1", "中" * (k // 3) + run + "中", run * 40]
    for t, a, b in zip(texts, tok.encode_batch(texts), live(texts)):
        assert a == b, (len(t.encode()), repr(t[-40:]))


@pytest.mark.parametrize("ignore_merges", [False, True])
def test_ignore_merges_both_values(tmp_path, ignore_merges):
    j = json.load(open(DEEPSEEK))
    j["model"]["ignore_merges"] = ignore_merges
    (tmp_path / "t.json").write_text(json.dumps(j))
    tok, rng = _policy().load_hf_tokenizer(str(tmp_path / "t.json")), random.Random(7)
    texts = json.load(open(os.path.join(GOLD, "deepseek_vectors.json")))["cases"]
    texts = [c["text"] for c in texts] + ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, 120))) for _ in range(200)]
    assert tok.encode_batch(texts) == _live(str(tmp_path / "t.json"))(texts)


def test_cap_tokens_is_total_bytes(tmp_path):
    """Without merges every byte is a token: cap_tokens = total bytes is exactly reached, one less is the capacity error, and the next
    call is answered."""
    j = json.load(open(DEEPSEEK))
    j["model"]["merges"] = []
    (tmp_path / "t.json").write_text(json.dumps(j))
    pol = _policy()
    tok = pol.load_hf_tokenizer(str(tmp_path / "t.json"), model="d")
    texts = ["中文テスト・アイ abc123456 !Hello", "١٢٣٤ ²³ 12345678", "x\x00\x01 ." * 20, "鿿" * 90]
    nbytes, want = sum(len(t.encode()) for t in texts), _live(str(tmp_path / "t.json"))(texts)
    assert sum(len(w) for w in want) == nbytes
    for cap, status in ((nbytes, _lib.SUCCESS), (nbytes - 1, _lib.INVALID_ARGUMENT)):
        out, toff = np.full(cap, 0xDEADBEEF, np.uint32), np.zeros(len(texts) + 1, np.uint32)
        assert _raw("smgx_tokenize_batch", pol, b"d", texts, out.ctypes.data_as(C.c_void_p), toff.ctypes.data_as(C.c_void_p), cap, None) == status
        if status == _lib.SUCCESS:
            assert [out[toff[i]:toff[i + 1]].tolist() for i in range(len(texts))] == want and toff[-1] == nbytes
    assert tok.encode_batch(texts) == want


def _submit(pol, model, texts):
    out, t = np.full(len(texts), -7, np.int32), C.c_uint64()
    data, offsets = TiktokenTokenizer._ragged(texts)
    pol._h.call("smgx_submit_text", model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(texts),
                out.ctypes.data_as(C.c_void_p), None, C.byref(t))
    return out, (data, offsets), t.value


def test_three_models_text_in_pick_equals_tokens_in_pick_and_oracle():
    """One policy holds "m-cl" (cl100k), "m-qwen" (the Qwen2+NFC fixture) and "m-ds" (the DeepSeek fixture), each with its own KV index.
    Per model the ids equal its reference (the oracle, or live `tokenizers`) and the text-in pick equals the tokens-in pick and the oracle
    policy's pick; smgx_submit_text calls of the three, interleaved over the stream lanes, pick the same."""
    bs, rng = 4, random.Random(2026)
    cfg = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=bs)
    pol = _policy(**cfg)
    r50k = json.load(open(os.path.join(GOLD, "r50k_vectors.json")))
    urls, models = synth.worker_urls(8), ["m-cl", "m-qwen", "m-ds"]
    fleets = {m: [BasicWorker(u, m) for u in urls] for m in models}
    pol.init_workers(sum(fleets.values(), []))
    loads = [rng.randint(0, 9) for _ in urls]
    words = "naïve café 中文 テスト・ケース 12345 it's 2024 the quick brown fox x=y+1 ١٢٣٤ ..abc !Hello ́".split(" ")
    system = [BOS + "system\n" + " ".join(rng.choice(words) for _ in range(30)) + " 1234567 it'S\n\n" for _ in range(6)]
    texts = [rng.choice(system) + USER + " ".join(rng.choice(words) for _ in range(rng.randint(1, 20))) + ASSISTANT
             for _ in range(200)] + [" ".join(rng.choice(words) for _ in range(12)) for _ in range(40)]
    mon, picks = pol.kv_event_monitor(bs), {}
    for shift, m in enumerate(models):
        if m == "m-cl":
            enc = bpe_ref.CoreBPE(bpe_ref.load_tiktoken_bpe(VOCAB), r50k["specials"], pattern=bpe_ref.CL100K_BASE_PATTERN)
            tok = pol.load_tiktoken_tokenizer(VOCAB, r50k["specials"], model=m, encoding="cl100k_base")
            encode = lambda ts, enc=enc: [enc.encode_with_special_tokens(t) for t in ts]   # noqa: E731
        else:
            path = QWEN2 if m == "m-qwen" else DEEPSEEK
            tok, encode = pol.load_hf_tokenizer(path, model=m), _live(path)
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


@pytest.mark.skipif(not os.environ.get("SMGX_REAL_DEEPSEEK_TOKENIZER_JSON"), reason="set SMGX_REAL_DEEPSEEK_TOKENIZER_JSON to a real "
                    "DeepSeek V2 / V3 / R1 tokenizer.json")
def test_real_deepseek_tokenizer_json():
    """A real file loads and matches live `tokenizers`."""
    path = os.environ["SMGX_REAL_DEEPSEEK_TOKENIZER_JSON"]
    try:
        tok = _policy().load_hf_tokenizer(path)
    except ValueError as e:
        pytest.fail(f"refused: {e}")
    rng = random.Random(5)
    texts = ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, 200))) for _ in range(400)]
    texts += ["Hello world! How are you today?", "  def main():\n\treturn 0", "日本語のテキスト・カタカナ", "🧑‍💻 ünïcödé ≠ ∑ 1234567"]
    assert tok.encode_batch(texts) == _live(path)(texts)
