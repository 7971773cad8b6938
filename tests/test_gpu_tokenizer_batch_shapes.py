"""Batch shapes of the GPU tokenizer through the C ABI, for every family the library loads: cl100k and r50k tiktoken files, byte-level
tokenizer.json of the Llama-3 and GPT-2 shapes, Qwen2 with NFC, Llama-2 (legacy ▁ normalizer and a Metaspace variant) and DeepSeek-V3.

- request counts around the scan's 1024-request tiles and past 65 535, the most CTAs a grid's y dimension holds;
- the text-in pick at max_batch (event-driven against the tokens-in pick and the oracle, tree mode against a policy fed the reference
  tokens), and a batch one over max_batch refused;
- offsets that do not start at 0, with bytes before offsets[0] that would change the result if a kernel read them;
- degenerate batches: all empty, one non-empty text at either end, runs of empty texts across the scan tiles, specials only, one 256 KiB
  text among short ones.

The references are live tiktoken / `tokenizers`, run once per family on its largest batch; smaller batches are prefixes of it."""
import ctypes as C
import itertools
import json
import os
import random
import unicodedata
import zlib

import numpy as np
import pytest

from oracle import bpe_ref, orc
from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy, _lib, synth
from smg_b200.policy import TiktokenTokenizer, _p
from tests.test_gpu_tokenizer_deepseek import ALPHABET as DEEPSEEK_ALPHABET
from tests.test_gpu_tokenizer_llama2 import ALPHABET as LLAMA2_ALPHABET, _variant
from tests.test_gpu_tokenizer_qwen2 import ALPHABET as QWEN2_ALPHABET
from tests.test_gpu_tokenizer_r50k import ALPHABET as R50K_ALPHABET

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
VOCAB = os.path.join(GOLD, "synth_vocab.tiktoken")
FAMILIES = ["cl100k", "r50k", "llama3", "gpt2", "qwen2", "llama2", "llama2-metaspace", "deepseek"]
HF = {"llama3": "hf_llama3_style_tokenizer.json", "gpt2": "hf_gpt2_style_tokenizer.json", "qwen2": "hf_qwen2_style_tokenizer.json",
      "llama2": "hf_llama2_style_tokenizer.json", "deepseek": "hf_deepseek_v3_style_tokenizer.json"}
ALPHABETS = {
    "cl100k": list("abcdefghij XYZ 0123\n\t\r'.,!?-_()<|>im_startend" + "éß你好\U0001f44b 　ſ"),
    "r50k": list(R50K_ALPHABET),
    "llama3": list("abcdefghij the quick XYZ 0123456789\n\t\r'.,!?-_(){}[]<|>eot_idbegin_of_text" + "éßüï你好世界\U0001f44b\U0001f30d ١٢٣"),
    "gpt2": list(R50K_ALPHABET),
    "qwen2": QWEN2_ALPHABET,
    "llama2": LLAMA2_ALPHABET,
    "llama2-metaspace": LLAMA2_ALPHABET,
    "deepseek": DEEPSEEK_ALPHABET,
}
COUNTS = [1, 1023, 1024, 1025, 65535, 65536, 65537]
LARGEST = {"cl100k": 131073, "qwen2": 131073}   # every other family: max(COUNTS)
PICK_N = {"cl100k": 131072}                     # text-in pick batches; every other family: 65536
BASES = [1, 4099, 1000003]
POISON = 0xDEADBEEF
BS = 4
CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=BS)
BRANCH = _lib.DecisionInfo.branch.offset


def _short_text(rng, alphabet, lens):
    """0-48 bytes of alphabet items (specials included)."""
    budget, out, used = rng.randint(0, 48), [], 0
    while True:
        k = rng.randrange(len(alphabet))
        if used + lens[k] > budget:
            return "".join(out)
        out.append(alphabet[k])
        used += lens[k]


def _flat(ids):
    toff = np.zeros(len(ids) + 1, np.uint32)
    np.cumsum([len(x) for x in ids], out=toff[1:])
    return np.fromiter(itertools.chain.from_iterable(ids), np.uint32, count=int(toff[-1])), toff


class Family:
    """One tokenizer family: how to load it, its live reference, and its largest batch of seeded short texts with the reference ids."""

    def __init__(self, name, tmp_path):
        self.name = name
        if name in ("cl100k", "r50k"):
            g = json.load(open(os.path.join(GOLD, "bpe_vectors.json" if name == "cl100k" else "r50k_vectors.json")))
            tiktoken = pytest.importorskip("tiktoken")
            enc = tiktoken.Encoding("synth-" + name, pat_str=g["pattern"] if name == "cl100k" else g["tiktoken_pattern"],
                                    mergeable_ranks=bpe_ref.load_tiktoken_bpe(VOCAB), special_tokens=g["specials"])
            self.specials = list(g["specials"])
            self.encode = lambda texts: enc.encode_batch(texts, num_threads=os.cpu_count() or 1, allowed_special="all")
            self.load = lambda pol, model: pol.load_tiktoken_tokenizer(VOCAB, g["specials"], model=model, encoding=name + "_base")
        else:
            path = _variant("metaspace-first-split", tmp_path) if name == "llama2-metaspace" else os.path.join(GOLD, HF[name])
            ref = pytest.importorskip("tokenizers").Tokenizer.from_file(path)
            self.specials = [a["content"] for a in json.load(open(path))["added_tokens"]]
            self.encode = lambda texts: [e.ids for e in ref.encode_batch(texts, add_special_tokens=False)]
            self.load = lambda pol, model: pol.load_hf_tokenizer(path, model=model)
        self.rng = random.Random(zlib.crc32(name.encode()))
        self.alphabet = ALPHABETS[name] + self.specials
        lens = [len(a.encode()) for a in self.alphabet]
        self.texts = [_short_text(self.rng, self.alphabet, lens) for _ in range(LARGEST.get(name, max(COUNTS)))]
        self.ids = self.encode(self.texts)
        self.data, self.offsets = TiktokenTokenizer._ragged(self.texts)
        self.flat, self.toff = _flat(self.ids)
        # system prompts for the text-in pick: they end with a special, so their tokens are a prefix of every request that starts with one
        self.system = [self.specials[k % len(self.specials)] + " ".join(self.texts[7 * k:7 * k + 4]) + self.specials[-1] for k in range(6)]
        self.system_ids = self.encode(self.system)
        self._pick = None

    def pick_batch(self):
        """System prompt + short text, PICK_N texts, with the reference ids (flat) and byte offsets."""
        if self._pick is None:
            rng = random.Random(zlib.crc32(b"pick-" + self.name.encode()))
            n = PICK_N.get(self.name, 65536)
            texts = [rng.choice(self.system) + self.texts[i % len(self.texts)] for i in range(n)]
            data, offsets = TiktokenTokenizer._ragged(texts)
            self._pick = (texts, data, offsets) + _flat(self.encode(texts))
        return self._pick


@pytest.fixture(scope="module")
def family(tmp_path_factory):
    made, tmp = {}, tmp_path_factory.mktemp("tokenizers")

    def get(name):
        if name not in made:
            made[name] = Family(name, tmp)
        return made[name]
    return get


@pytest.fixture(scope="module")
def tok_policy(family):
    """One policy with every family loaded as its own model; → (policy, growth by family)."""
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0))
    loaded = {}

    def get(name):
        if name not in loaded:
            loaded[name] = family(name).load(pol, name).growth
        return pol, loaded[name]
    yield get
    pol.close()


def _tokenize(pol, model, data, offsets, n, growth):
    """smgx_tokenize_batch on texts 0..n-1 of (data, offsets); the output past the written tokens must stay untouched."""
    cap = growth * int(offsets[n] - offsets[0]) + 1
    out, toff = np.full(cap + 16, POISON, np.uint32), np.full(n + 1, POISON, np.uint32)
    pol._h.call("smgx_tokenize_batch", model, _p(data), _p(offsets), n, _p(out), _p(toff), cap)
    assert (out[toff[n]:] == POISON).all()
    return out[:toff[n]], toff


def _check(got, want_flat, want_toff, what):
    flat, toff = got
    assert toff.size == want_toff.size and toff[0] == 0, what
    bad = np.flatnonzero(toff != want_toff)
    assert bad.size == 0, (what, "first wrong token offset at request", int(bad[0]) if bad.size else None)
    assert np.array_equal(flat, want_flat), (what, "ids differ")


# ---- a. request counts ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n", [(f, n) for f in FAMILIES for n in COUNTS + ([LARGEST[f]] if f in LARGEST else [])])
def test_request_counts(family, tok_policy, name, n):
    """n texts in one smgx_tokenize_batch call: below, at and past the scan's 1024-request tiles and the 65 535 requests one grid
    dimension holds (the per-request kernels fold the request index over two)."""
    f = family(name)
    pol, growth = tok_policy(name)
    _check(_tokenize(pol, name.encode(), f.data, f.offsets, n, growth), f.flat[:f.toff[n]], f.toff[:n + 1], (name, n))


# ---- b. text-in pick at max_batch -------------------------------------------------------------------------------------------------
def _pick_policy(f, max_batch=0, indexer=True):
    """Policy with f loaded as model "m" on 8 workers; with `indexer`, an event indexer holding the system prompts on two workers each
    and the oracle policy in the same state.  → (policy, workers, growth, oracle policy or None)."""
    rng = random.Random(77)
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **CFG), max_batch=max_batch)
    growth = f.load(pol, "m").growth
    urls = synth.worker_urls(8)
    ws = [BasicWorker(u, "m") for u in urls]
    pol.init_workers(ws)
    loads = [rng.randint(0, 9) for _ in urls]
    for w, l in zip(ws, loads):
        w.set_load(l)
    op = None
    if indexer:
        mon, oix = pol.kv_event_monitor(BS), orc.PositionalIndexer(8)
        ix = mon.create_indexer("m", 8)
        op = orc.CacheAwarePolicy(eviction_interval_secs=0, **CFG)
        op.set_workers(urls, models=["m"] * 8)
        op.attach_indexer("m", oix)
        op.set_kv_event_monitor(True)
        op.set_state(loads, [1] * 8, [1] * 8)
        for u in urls:
            assert ix.intern_worker(u) == oix.intern_worker(u)
        seq = 1
        for k, ids in enumerate(f.system_ids):
            hs = orc.compute_request_content_hashes(ids, BS)
            blocks = [(seq + i, hs[i]) for i in range(len(ids) // BS)]
            seq += len(blocks)
            for w in (k % 8, (k + 3) % 8):
                ix.apply_stored(w, blocks)
                oix.apply_stored(w, blocks)
        pol.set_kv_event_monitor(mon)
    pol._push_fleet(ws)
    return pol, ws, growth, op


def _select_text(pol, data, offsets, n, growth):
    """Raw smgx_select_batch_text → (status, picks, branches, (ids, token offsets))."""
    cap = growth * int(offsets[n] - offsets[0]) + 1
    out, info = np.full(n, -7, np.int32), (_lib.DecisionInfo * n)()
    toks, toff = np.full(cap + 16, POISON, np.uint32), np.full(n + 1, POISON, np.uint32)
    st = pol._h.L.smgx_select_batch_text(pol._h.p, b"m", _p(data), _p(offsets), n, _p(out), C.cast(info, C.c_void_p), _p(toks), _p(toff),
                                         cap, None)
    br = np.frombuffer(info, np.uint8).reshape(n, C.sizeof(_lib.DecisionInfo))[:, BRANCH].copy()
    return st, out, br, (toks[:toff[n]] if st == _lib.SUCCESS else None, toff)


def _submit_text(pol, data, offsets, n):
    out, t = np.full(n, -7, np.int32), C.c_uint64()
    pol._h.call("smgx_submit_text", b"m", _p(data), _p(offsets), n, _p(out), None, C.byref(t))
    return out, t.value


def _tokens_in_and_oracle(pol, ws, op, flat, toff):
    idx_tok, _ = pol.select_worker_batch(ws, tokens=flat, offsets=toff, want_info=False)
    want, br, _, _ = op.select_batch_tokens(flat, toff.astype(np.uint64))
    assert np.array_equal(idx_tok, want)
    return want, np.asarray(br)


@pytest.mark.parametrize("name", ["cl100k", "qwen2", "llama2"])
def test_text_in_pick_at_max_batch(family, name):
    """With the default max_batch (65 536), a full batch picks as the tokens-in pick on the reference tokens and as the oracle; the
    returned tokens are the reference; two smgx_submit_text batches of 65 536 in flight pick the same; 65 537 texts are refused with
    SMGX_INVALID_ARGUMENT and the next call is answered."""
    f = family(name)
    n = 65536
    _, data, offsets, flat, toff = f.pick_batch()
    pol, ws, growth, op = _pick_policy(f)
    want, want_br = _tokens_in_and_oracle(pol, ws, op, flat[:toff[n]], toff[:n + 1])
    st, out, br, toks = _select_text(pol, data, offsets, n, growth)
    assert st == _lib.SUCCESS
    _check(toks, flat[:toff[n]], toff[:n + 1], name)
    assert np.array_equal(out, want) and np.array_equal(br, want_br)
    assert (br == 2).sum() > n // 4   # most requests hit a cached system prompt
    assert pol._h.L.smgx_pipeline_depth(pol._h.p) >= 2
    rev = TiktokenTokenizer._ragged([f.pick_batch()[0][i] for i in range(n - 1, -1, -1)])
    (a, ta), (b, tb) = _submit_text(pol, data, offsets, n), _submit_text(pol, rev[0], rev[1], n)
    pol._h.call("smgx_wait", ta)
    pol._h.call("smgx_wait", tb)
    assert np.array_equal(a, want) and np.array_equal(b, want[::-1])
    over = np.append(offsets[:n + 1], offsets[n])   # one more (empty) text
    assert _select_text(pol, data, over, n + 1, growth)[0] == _lib.INVALID_ARGUMENT
    st, out, _, _ = _select_text(pol, data, offsets, n, growth)
    assert st == _lib.SUCCESS and np.array_equal(out, want)
    pol.close()


def test_text_in_pick_of_131072_with_max_batch_131072(family):
    f = family("cl100k")
    texts, data, offsets, flat, toff = f.pick_batch()
    n = len(texts)
    assert n == 131072
    pol, ws, growth, op = _pick_policy(f, max_batch=n)
    want, want_br = _tokens_in_and_oracle(pol, ws, op, flat, toff)
    st, out, br, toks = _select_text(pol, data, offsets, n, growth)
    assert st == _lib.SUCCESS
    _check(toks, flat, toff, "cl100k")
    assert np.array_equal(out, want) and np.array_equal(br, want_br)
    pol.close()


def test_tree_mode_text_in_pick_at_max_batch(family):
    """Without an event indexer the text-in pick walks the approximate token tree on the tokens it made: two rounds of 65 536 Qwen2 texts
    pick as a second policy in the same state that is fed the reference tokens (the second round sees the first round's inserts)."""
    f = family("qwen2")
    _, data, offsets, flat, toff = f.pick_batch()
    n = 65536
    pol, ws, growth, _ = _pick_policy(f, indexer=False)
    twin, ws2, _, _ = _pick_policy(f, indexer=False)
    for rnd in range(2):
        st, out, br, toks = _select_text(pol, data, offsets, n, growth)
        assert st == _lib.SUCCESS
        _check(toks, flat[:toff[n]], toff[:n + 1], ("qwen2 tree", rnd))
        idx, info = twin.select_worker_batch(ws2, tokens=flat[:toff[n]], offsets=toff[:n + 1])
        assert np.array_equal(out, idx), rnd
        assert np.array_equal(br, np.asarray([i.branch for i in info], np.uint8)), rnd
    pol.close()
    twin.close()


# ---- c. offsets that do not start at 0 --------------------------------------------------------------------------------------------
def _long_texts():
    """Texts whose NFC segments decompose to more than 32 code points (the long-segment kernel), ▁ and space stretches, and runs across
    the 256-byte chunks."""
    return ["\u0301" * 40 + "y", "x" + "\u0323\u0301\u0308" * 20, "a" * 250 + "\u0301" * 40 + " b", unicodedata.normalize("NFD", "é") * 200,
            "▁" * 300 + "a", " " * 300 + "b", "中" * 100 + " 1234", "<>" * 150]


def _poisons(f):
    """(bytes just before offsets[0], text 0).  Text 0 starts with what would continue those bytes, so its tokens change if a kernel reads
    behind offsets[0] or loses its start-of-request rule: the pre-tokenizer's anchor test at the first byte (`gi == beg`), the NFC segment
    start (`i == beg`), the ▁ prepend (`i == beg`), the special matcher."""
    assert f.specials[0].endswith(">")   # one ASCII byte: text 0 completes the cut special
    return [(b"\xf0\xc3\xe4", "ab 12"),                      # lead bytes of a 4-, 2- and 3-byte sequence; a letter after them is no anchor
            ("\u0301".encode(), "\u0301x"),                  # a combining mark; a mark after it starts no NFC segment
            (f.specials[0].encode()[:-1], ">abc"),           # a special cut one byte short
            ("▁".encode(), " x▁y")]                          # ▁; a space after it is no anchor, and no ▁ is prepended


@pytest.mark.parametrize("name", FAMILIES)
def test_offsets_not_starting_at_zero(family, name):
    """3 000 texts at base 1, 4 099 and 1 000 003 of a larger buffer, with offsets shifted by base.  The bytes in front of base are UTF-8
    lead bytes, a combining mark, a special cut one byte short, or ▁, and text 0 continues them (_poisons).  smgx_tokenize_batch,
    smgx_select_batch_text and smgx_submit_text give what the zero-based call gives, and that is the reference."""
    f = family(name)
    rest = [f.system[k % 6] + t for k, t in enumerate(f.texts[:1500])] + f.texts[1500:2991] + _long_texts()
    poisons = _poisons(f)
    want_rest, want_first = f.encode(rest), f.encode([t for _, t in poisons])
    pol, ws, growth, _ = _pick_policy(f)
    for (junk, first), first_ids in zip(poisons, want_first):
        texts = [first] + rest
        assert len(texts) == 3000
        want = _flat([first_ids] + want_rest)
        data, offsets = TiktokenTokenizer._ragged(texts)
        n = len(texts)
        _check(_tokenize(pol, b"m", data, offsets, n, growth), *want, (name, 0, junk))
        st, out0, br0, toks = _select_text(pol, data, offsets, n, growth)
        assert st == _lib.SUCCESS
        _check(toks, *want, (name, "select", 0, junk))
        sub0, t = _submit_text(pol, data, offsets, n)
        pol._h.call("smgx_wait", t)
        assert np.array_equal(sub0, out0)
        for base in BASES:
            buf = np.empty(base + data.size, np.uint8)
            buf[:base] = np.frombuffer((junk * (base // len(junk) + 1))[-base:], np.uint8)   # ends with the whole of junk
            buf[base:] = data
            shifted = offsets + np.uint32(base)
            what = (name, base, junk)
            _check(_tokenize(pol, b"m", buf, shifted, n, growth), *want, what)
            st, out, br, toks = _select_text(pol, buf, shifted, n, growth)
            assert st == _lib.SUCCESS, what
            _check(toks, *want, what)
            assert np.array_equal(out, out0) and np.array_equal(br, br0), what
            sub, t = _submit_text(pol, buf, shifted, n)
            pol._h.call("smgx_wait", t)
            assert np.array_equal(sub, out0), what
    pol.close()


# ---- d. degenerate batches --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FAMILIES)
def test_all_empty_texts(tok_policy, name):
    """70 000 empty texts (no pre-tokenizer or BPE launch, only the scan and the compaction), at offset 0 and at offset 3."""
    pol, growth = tok_policy(name)
    n = 70000
    for base in (0, 3):
        data = np.frombuffer(b"\xe4\xb8\xad\xcc", np.uint8).copy()
        got = _tokenize(pol, name.encode(), data, np.full(n + 1, base, np.uint32), n, growth)
        _check(got, np.zeros(0, np.uint32), np.zeros(n + 1, np.uint32), (name, base))


@pytest.mark.parametrize("name", FAMILIES)
def test_one_non_empty_text_first_or_last(family, tok_policy, name):
    """65 537 texts of which only the first, or only the last, is non-empty."""
    f = family(name)
    pol, growth = tok_policy(name)
    k = max(range(1000), key=lambda i: len(f.ids[i]))
    data = np.frombuffer(f.texts[k].encode(), np.uint8).copy()
    L, n = data.size, 65537
    ids = np.asarray(f.ids[k], np.uint32)
    first = np.full(n + 1, L, np.uint32)
    first[0] = 0
    last = np.zeros(n + 1, np.uint32)
    last[n] = L
    _check(_tokenize(pol, name.encode(), data, first, n, growth), ids, np.where(np.arange(n + 1) == 0, 0, ids.size).astype(np.uint32), name)
    _check(_tokenize(pol, name.encode(), data, last, n, growth), ids, np.where(np.arange(n + 1) == n, ids.size, 0).astype(np.uint32), name)


@pytest.mark.parametrize("name", FAMILIES)
def test_runs_of_empty_texts_across_scan_tiles(family, tok_policy, name):
    """6 000 texts where [1000, 2500), [3000, 4500) and [5500, 6000) are empty: runs of 1 500 that straddle the scan's 1024-request tiles."""
    f = family(name)
    pol, growth = tok_policy(name)
    empty = set(range(1000, 2500)) | set(range(3000, 4500)) | set(range(5500, 6000))
    texts = ["" if i in empty else f.texts[i] for i in range(6000)]
    data, offsets = TiktokenTokenizer._ragged(texts)
    want = _flat([[] if i in empty else f.ids[i] for i in range(6000)])
    _check(_tokenize(pol, name.encode(), data, offsets, len(texts), growth), *want, name)


@pytest.mark.parametrize("name", FAMILIES)
def test_specials_only(family, tok_policy, name):
    """65 536 texts that are each exactly one special token."""
    f = family(name)
    pol, growth = tok_policy(name)
    one = f.encode(f.specials)
    texts = [f.specials[i % len(f.specials)] for i in range(65536)]
    data, offsets = TiktokenTokenizer._ragged(texts)
    want = _flat([one[i % len(f.specials)] for i in range(65536)])
    _check(_tokenize(pol, name.encode(), data, offsets, len(texts), growth), *want, name)


@pytest.mark.parametrize("name", FAMILIES)
def test_one_256kib_text_among_short_ones(family, tok_policy, name):
    """One text of 256 KiB at request 40 000 of 65 536 (the others short): every request's grid row spans the long text's chunks."""
    f = family(name)
    pol, growth = tok_policy(name)
    rng, parts, used = random.Random(256), [], 0
    while True:
        a = rng.choice(f.alphabet)
        if used + len(a.encode()) > 262144:
            break
        parts.append(a)
        used += len(a.encode())
    big = "".join(parts) + "x" * (262144 - used)
    assert len(big.encode()) == 262144
    texts = f.texts[:40000] + [big] + f.texts[40000:65535]
    data, offsets = TiktokenTokenizer._ragged(texts)
    want = _flat(f.ids[:40000] + f.encode([big]) + f.ids[40000:65535])
    _check(_tokenize(pol, name.encode(), data, offsets, len(texts), growth), *want, name)
