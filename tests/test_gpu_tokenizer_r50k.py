"""GPU parity of the GPT-2 (r50k) pre-tokenizer: tiktoken encodings r50k_base / p50k_base / p50k_edit and GPT-2-style tokenizer.json files
through the C ABI, against the golden vectors (tests/golden/gen_r50k_golden.py), the oracle with the r50k pattern, live tiktoken and
live `tokenizers`; window and piece-length edges; the text-in pick; and a cl100k and an r50k model side by side in one policy."""
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

from oracle import bpe_ref, orc
from smg_b200 import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
VOCAB = os.path.join(GOLD, "synth_vocab.tiktoken")
ALPHABET = ("abcdefghij XYZ 0123456789 sdmtlvrSDMTLVRe '''\n\n\r\t\t  .,!?-_()<|>im_startend" + "\x1c\x1d\x1e\x1f\x85\xa0᠎​　﻿́"
            + "½Ⅰ١٢éß你好\U0001f44b")


def _gold():
    return json.load(open(os.path.join(GOLD, "r50k_vectors.json")))


def _policy_and_tok(encoding="r50k_base", **cfg):
    from smg_b200 import CacheAwareConfig, CacheAwarePolicy
    g = _gold()
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **cfg))
    return pol, pol.load_tiktoken_tokenizer(VOCAB, g["specials"], encoding=encoding), g


def _oracle(g, pattern=None):
    return bpe_ref.CoreBPE(bpe_ref.load_tiktoken_bpe(VOCAB), g["specials"], pattern=pattern or g["pattern"])


@pytest.mark.parametrize("encoding", ["r50k_base", "p50k_base", "p50k_edit"])
def test_r50k_golden_vectors_on_gpu(encoding):
    pol, tok, g = _policy_and_tok(encoding)
    got = tok.encode_batch([c["text"] for c in g["cases"]])
    for c, ids in zip(g["cases"], got):
        assert ids == c["ids"], repr(c["text"][:80])
    assert tok.encode("") == [] and tok.encode("<|endoftext|>") == [g["specials"]["<|endoftext|>"]]


def test_random_text_vs_oracle_and_live_tiktoken():
    pol, tok, g = _policy_and_tok()
    enc = _oracle(g)
    rng = random.Random(505)
    texts = ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, 400))) for _ in range(1500)]
    texts += ["word " * 500, "1" * 3000, " " * 2000 + "end", "\n".join("line %d: it's the quick brown fox's 2024" % i for i in range(200))]
    got = tok.encode_batch(texts)
    for t, ids in zip(texts, got):
        assert ids == enc.encode_with_special_tokens(t), repr(t[:80])
    tiktoken = pytest.importorskip("tiktoken")
    live = tiktoken.Encoding("synth_r50k", pat_str=g["tiktoken_pattern"], mergeable_ranks=bpe_ref.load_tiktoken_bpe(VOCAB), special_tokens=g["specials"])
    for t, ids in zip(texts, got):
        assert ids == live.encode(t, allowed_special="all"), repr(t[:80])


def _hf_tok():
    from smg_b200 import CacheAwareConfig, CacheAwarePolicy
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0))
    return pol, pol.load_hf_tokenizer(os.path.join(GOLD, _gold()["hf"]["fixture"]))


def test_hf_gpt2_fixture_matches_its_goldens():
    hf = _gold()["hf"]
    pol, tok = _hf_tok()
    for t, ids, want in zip(hf["texts"], tok.encode_batch(hf["texts"]), hf["ids"]):
        assert ids == want, repr(t[:80])


def test_hf_gpt2_fixture_matches_live_tokenizers_on_random_texts():
    tokenizers = pytest.importorskip("tokenizers")
    pol, tok = _hf_tok()
    ref = tokenizers.Tokenizer.from_file(os.path.join(GOLD, _gold()["hf"]["fixture"]))
    rng = random.Random(506)
    alphabet = ALPHABET + "the quick brown fox <|endoftext|>"
    texts = ["".join(rng.choice(alphabet) for _ in range(rng.randint(0, 400))) for _ in range(800)]
    texts += ["<|endoftext|>" + "hello world " * 50 + "<|endoftext|>", "don't DON'T I'LL we'Ve 'S", "   \n\n  \n x  \n", "12345678901234567890"]
    got = tok.encode_batch(texts)
    want = [e.ids for e in ref.encode_batch(texts, add_special_tokens=False)]
    for t, a, b in zip(texts, got, want):
        assert a == b, repr(t[:80])


def test_window_edges_vs_oracle():
    """The kernel classifies 256-byte windows of a request; pieces that cross a window edge, and anchors right at one, take the
    global-memory matcher and the global anchor test."""
    pol, tok, g = _policy_and_tok()
    enc = _oracle(g)
    texts = []
    for k in list(range(248, 264)) + list(range(506, 518)):
        texts += ["a" * k + "bcd efg", "x" * (k - 1) + " 12345 6", "1" * k + "234 x", "-" * k + "=+ !", " " * k + "  x", " " * k + "\t\tx",
                  "z" * (k - 1) + "'s 'll", "z" * (k - 2) + "'ve", "q" * (k - 1) + " 1", "q" * (k - 2) + " 1999", "w" * (k - 1) + "!'s",
                  "w" * (k - 2) + "''s", "y" * (k - 1) + "<|endoftext|> z", "y" * k + "<|endoftext|>'s", "y" * (k - 2) + "  <|im_end|>\n",
                  "é" * (k // 2) + "'s" + "1" * 20, "\n" * k + "\n\nx", "a" * (k - 3) + "\xa0\xa0x"]
    got = tok.encode_batch(texts)
    for t, ids in zip(texts, got):
        assert ids == enc.encode_with_special_tokens(t), (len(t.encode()), repr(t[-40:]))


def test_piece_length_classes_vs_oracle():
    """r50k's unbounded digit runs and space-led punctuation runs reach every merge kernel (≤ 15 bytes, 16-32, 33-256, > 256)."""
    pol, tok, g = _policy_and_tok()
    enc = _oracle(g)
    rng = random.Random(507)
    texts = []
    for k in list(range(1, 70)) + [100, 127, 128, 129, 200, 255, 256, 257, 300, 1000]:
        texts += [" " * k + "x", "-" * k, " " + "!" * k, "1" * k, " " + "9" * k, "ab" * k, "".join(rng.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(k)),
                  "".join(rng.choice("0123456789") for _ in range(k)), "".join(rng.choice("éßü你好") for _ in range(k)), "=" * k + "\n" * (k % 5),
                  "a" * k + " " + "b" * k, "\n" * k + "x"]
    got = tok.encode_batch(texts)
    for t, ids in zip(texts, got):
        assert ids == enc.encode_with_special_tokens(t), (len(t), repr(t[:40]))


def _submit_text(pol, jobs):
    """smgx_submit_text for every (model key, texts) job with as many in flight as there are stream lanes → the pick arrays."""
    from smg_b200.policy import TiktokenTokenizer
    depth = pol._h.L.smgx_pipeline_depth(pol._h.p)
    bufs, tickets = [], []
    for model, part in jobs:
        if len(tickets) >= depth:
            pol._h.call("smgx_wait", tickets[len(tickets) - depth])
        data, offsets = TiktokenTokenizer._ragged(part)
        out = np.full(len(part), -7, np.int32)
        t = C.c_uint64()
        pol._h.call("smgx_submit_text", model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(part),
                    out.ctypes.data_as(C.c_void_p), None, C.byref(t))
        bufs.append((data, offsets, out))
        tickets.append(t.value)
    for t in tickets[-depth:]:
        pol._h.call("smgx_wait", t)
    return [b[2] for b in bufs]


def test_two_models_text_in_pick_equals_tokens_in_pick_and_oracle():
    """One policy holds model "m-cl" (cl100k) and "m-r50k" (r50k) over the same vocabulary, each with its own KV index.  Per model: the
    token ids equal its own oracle, and the text-in pick equals the tokens-in pick and the oracle policy's pick.  Submissions of the two
    models interleaved over the stream lanes (smgx_submit_text) pick the same."""
    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
    bs, g, rng = 4, _gold(), random.Random(509)
    cfg = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=bs)
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **cfg))
    models = {"m-cl": ("cl100k_base", bpe_ref.CL100K_BASE_PATTERN), "m-r50k": ("r50k_base", g["pattern"])}
    urls = synth.worker_urls(8)
    fleets = {m: [BasicWorker(u, m) for u in urls] for m in models}
    pol.init_workers(fleets["m-cl"] + fleets["m-r50k"])
    loads = [rng.randint(0, 9) for _ in urls]
    lines = [c["text"] for c in g["cases"] if len(c["ids"]) >= 12 and "<|" not in c["text"]]
    # system prompts the two patterns split differently: space-led digit runs, apostrophes, newline runs
    system = ["<|im_start|>system\n" + rng.choice(lines) + " 2024 1234567 it'S !'s\n\n\nx<|im_end|>\n" for _ in range(6)]
    texts = [rng.choice(system) + "<|im_start|>user\n" + rng.choice(lines) + "<|im_end|>\n" for _ in range(200)] + [rng.choice(lines) for _ in range(56)]
    mon = pol.kv_event_monitor(bs)
    picks, encs = {}, {}
    for shift, (m, (encoding, pattern)) in enumerate(models.items()):
        tok = pol.load_tiktoken_tokenizer(VOCAB, g["specials"], model=m, encoding=encoding)
        encs[m] = enc = _oracle(g, pattern)
        ix = mon.create_indexer(m, 8)
        op = orc.CacheAwarePolicy(eviction_interval_secs=0, **cfg)
        op.set_workers(urls, models=[m] * 8)
        oix = orc.PositionalIndexer(8)
        op.attach_indexer(m, oix)
        op.set_kv_event_monitor(True)
        for u in urls:
            assert ix.intern_worker(u) == oix.intern_worker(u)
        seq = 1
        for k, sp in enumerate(system):   # the two models cache the prompts on different workers
            ids = enc.encode_with_special_tokens(sp)
            hs = orc.compute_request_content_hashes(ids, bs)
            blocks = [(seq + i, hs[i]) for i in range(len(ids) // bs)]
            seq += len(blocks)
            for w in ((k + 4 * shift) % 8, (k + 4 * shift + 3) % 8):
                ix.apply_stored(w, blocks)
                oix.apply_stored(w, blocks)
        for w, l in zip(fleets[m], loads):
            w.set_load(l)
        op.set_state(loads, [1] * 8, [1] * 8)
        pol.set_kv_event_monitor(mon)
        idx_text, _, toks = pol.select_worker_batch_text(fleets[m], texts)
        assert toks == [enc.encode_with_special_tokens(t) for t in texts] == tok.encode_batch(texts), m
        idx_tok, _ = pol.select_worker_batch(fleets[m], toks)
        flat = np.concatenate([np.asarray(t, np.uint32) for t in toks])
        offs = np.zeros(len(toks) + 1, np.uint64); np.cumsum([len(t) for t in toks], out=offs[1:])
        want, br, _, _ = op.select_batch_tokens(flat, offs)
        assert np.array_equal(idx_text, idx_tok) and np.array_equal(idx_text, want), m
        assert (np.asarray(br) == 2).sum() > 100, m   # most requests hit a cached system prompt
        picks[m] = idx_text
    assert any(encs["m-cl"].encode_with_special_tokens(t) != encs["m-r50k"].encode_with_special_tokens(t) for t in texts)
    assert not np.array_equal(picks["m-cl"], picks["m-r50k"])
    keys = {m: pol._push_fleet(fleets[m]) for m in models}
    order = ["m-cl", "m-r50k"] * 4
    outs = _submit_text(pol, [(keys[m], texts[i // 2::4]) for i, m in enumerate(order)])
    for i, (m, out) in enumerate(zip(order, outs)):
        assert np.array_equal(out, picks[m][i // 2::4]), (m, i)
