"""Long requests through the approximate-tree walks (token tree and string tree), against the oracle and a closed form.

Both walk kernels process a request in fixed-size pieces: the token walk stages 512 tokens per warp and compares labels 256 tokens
per round (two 128-token halves), reports at most kPathCap = 32 path nodes and stages scalar when the request is not 16 B aligned;
the string walk stages 4080 usable bytes per warp, compares labels 512 B per round from any alignment, steps back over continuation
bytes after a mismatch and counts matched chars of a partial edge in 2048 B chunks.  The cases here put a mismatch, a request end
or a multi-byte char on each of those boundaries, build paths deeper than 32 and 255 nodes, and start requests at every alignment.

Every case has two independent answers: the oracle (one request at a time for SEQUENTIAL, one snapshot batch for SNAPSHOT), and,
for trees built by inserts only, a closed form — the longest common char prefix with any inserted text for the string tree, and
16·⌊lcp / 16⌋ over the page-aligned part of any inserted sequence for the token tree.  The tests without the gpu mark check the
generators (each case sits on the boundary its name gives) and that the oracle equals the closed form."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth

PAGE = 16
CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=16)
INSERTING = {1, 4, 5}     # imbalanced_min_load, tree_match, tree_min_load: the branches that insert the request (cache_aware.rs:396, :868)


# =====================================================================================================================
# closed forms
# =====================================================================================================================
def _lcp(a, b):
    n = min(len(a), len(b))
    if n == 0:
        return 0
    d = np.flatnonzero(np.asarray(a[:n], np.int64) != np.asarray(b[:n], np.int64))
    return int(d[0]) if d.size else n


def token_closed_form(inserted, q):
    """matched tokens of q against a token tree built only by inserting `inserted`: whole pages of the longest common prefix."""
    best = 0
    for s in inserted:
        best = max(best, _lcp(s[: len(s) // PAGE * PAGE], q) // PAGE * PAGE)
    return best


def text_closed_form(inserted, q):
    """matched chars of q against a string tree built only by inserting `inserted`."""
    return max([len(os.path.commonprefix([s, q])) for s in inserted] + [0])


# =====================================================================================================================
# token-tree cases
# =====================================================================================================================
S_PAGES = 96                                   # 1 536 tokens: 3 windows of 512, 6 rounds of 256
BRANCH_TOKEN = 100000                          # branch pages use ids ≥ this; S and its mutations stay below


def _base_tokens():
    return np.random.default_rng(11).integers(1, 50000, size=S_PAGES * PAGE, dtype=np.uint32)


S = _base_tokens()
TOKEN_SHAPES = {"one_node": [], "split_at_page_5": [5], "chain": [1, 3, 17, 33, 40, 64]}
# mismatch positions, by the boundary each one sits on
TOKEN_MISMATCH = {
    "quad": [0, 1, 2, 3],                      # every residue mod 4
    "page": [15, 16, 17],                      # page edge
    "label80": [79, 80, 81],                   # the label that starts at token 80 after the split at page 5
    "half": [127, 128],                        # the two 128-token halves of a round
    "round": [255, 256, 257],
    "window": [511, 512, 513, 1023, 1024],
    "last": [S_PAGES * PAGE - 1],
}


def _branch_page(p):
    return np.arange(BRANCH_TOKEN + 16 * p, BRANCH_TOKEN + 16 * p + PAGE, dtype=np.uint32)


def token_inserts(shape):
    """[(sequence, tenant)]: S, then one branch per split page (splits S's node there)."""
    out = [(S, "http://w0")]
    for i, p in enumerate(TOKEN_SHAPES[shape]):
        out.append((np.concatenate([S[: p * PAGE], _branch_page(p)]), f"http://w{1 + i % 3}"))
    return out


def _tail(n, seed):
    return np.random.default_rng(1000 + seed).integers(60000, 90000, size=n, dtype=np.uint32)


def token_cases():
    """[(name, query, kind, at)]"""
    cases = []
    for where, ps in TOKEN_MISMATCH.items():
        for p in ps:
            q = S.copy()
            q[p] = S[p] + 50000
            cases.append((f"mismatch_{where}@{p}", q, "mismatch", p))
            cases.append((f"stop_{where}@{p}", S[:p].copy(), "stop", p))
    cases.append(("stop_full@1536", S.copy(), "stop", len(S)))
    for k in (1, 3, 33):
        cases.append((f"extend_{k}_pages", np.concatenate([S, _tail(k * PAGE, k)]), "extend", len(S)))
    for r in range(1, 16):
        cases.append((f"ragged_tail_{r}", np.concatenate([S, _tail(r, 100 + r)]), "ragged", r))
    for p, r in ((256, 5), (513, 11), (1024, 15)):
        q = np.concatenate([S, _tail(r, 200 + r)])
        q[p] = S[p] + 50000
        cases.append((f"mismatch@{p}_ragged_tail_{r}", q, "mismatch", p))
    return cases


TOKEN_CASES = token_cases()


def _on_boundary(where, p):
    near = lambda unit: any(abs(p - k * unit) <= 1 for k in range(1, 8))
    return {"quad": p < 4, "page": p % PAGE in (15, 0, 1) and p < 32, "label80": abs(p - 80) <= 1,
            "half": p % 256 in (127, 128), "round": near(256), "window": near(512), "last": p == len(S) - 1}[where]


# =====================================================================================================================
# string-tree cases
# =====================================================================================================================
ASCII = "abcdefghijklmnopqrstuvwxyz ABCDEFGHIJ,.0123456789"
TWO = "éñüßçøåж"           # 2-byte
THREE = "中文字日本語€調度"   # 3-byte
FOUR = "🔥😀🚀𝄞👋🌍"          # 4-byte


def mixed_text(seed, n_bytes, pins=None):
    """Seeded text of about n_bytes UTF-8 bytes, mixed scripts; pins {byte offset: char} puts that char at that byte."""
    pins = pins or {}
    r = random.Random(seed)
    out, pos = [], 0
    while pos < n_bytes:
        if pos in pins:
            c = pins[pos]
        else:
            x = r.random()
            c = r.choice(ASCII if x < 0.55 else TWO if x < 0.7 else THREE if x < 0.88 else FOUR)
            if any(pos < p < pos + len(c.encode()) for p in pins):
                c = r.choice(ASCII)
        out.append(c)
        pos += len(c.encode())
    return "".join(out)


# (first byte, char): multi-byte chars straddling the lane (16), round (512), char-count chunk (2048) and window (4080 / 4081,
# 8160) boundaries; 509 is an ASCII char boundary for the split shape
STRADDLES = {"lane_15/16": (15, "é"), "round_511/512": (510, "🔥"), "chunk_2047/2048": (2046, "中"),
             "window_4079/4080/4081": (4078, "🚀"), "window_8159/8160": (8157, "😀")}
STRADDLE_BOUNDARIES = {"lane_15/16": [16], "round_511/512": [512], "chunk_2047/2048": [2048], "window_4079/4080/4081": [4080, 4081],
                       "window_8159/8160": [8160]}
T = mixed_text(7, 12 * 1024, {0: "T", 509: "k", **{b: c for b, c in STRADDLES.values()}})
TB = T.encode()
SPLITS = [509, 4078]              # T[:k] + "Ω" splits T's node at byte k (not 16-aligned; 4078 is 2 bytes before the window end)


def _char_at(b):
    """index of the char that starts at byte b of T"""
    assert TB[b] & 0xC0 != 0x80
    return len(TB[:b].decode())


def _swap(q_bytes, b, c_new):
    c_old = TB[b:].decode("utf-8", "ignore")[0]
    return (q_bytes[:b] + c_new.encode() + q_bytes[b + len(c_old.encode()):]).decode()


def text_cases():
    """[(name, query, kind, byte)]: kind "last" / "lead" = the straddling char replaced by one differing only in its last / lead
    byte; "end" = the query ends at that byte; "extend" = T plus more; "full" = T."""
    cases = []
    for name, (b, c) in STRADDLES.items():
        cp, n = ord(c), len(c.encode())
        cases.append((f"last_byte_{name}", _swap(TB, b, chr(cp + 1)), "last", b))
        cases.append((f"lead_byte_{name}", _swap(TB, b, chr(cp ^ (1 << (6 * (n - 1))))), "lead", b))
        cases.append((f"end_before_{name}", TB[:b].decode(), "end", b))
        cases.append((f"end_after_{name}", TB[:b + n].decode(), "end", b + n))
    for b in (32, 1024, 6000):
        while TB[b] & 0xC0 == 0x80:
            b += 1
        cases.append((f"end_at_{b}", TB[:b].decode(), "end", b))
    cases.append(("full", T, "full", len(TB)))
    cases.append(("extend_short", T + " and then 🔥 more", "extend", len(TB)))
    cases.append(("extend_long", T + mixed_text(8, 5000), "extend", len(TB)))
    return cases


TEXT_CASES = text_cases()
ARENA_RESIDUES = list(range(16))


def text_shape_inserts(shape):
    """[(text, tenant)] for "one_node", "split_<k>" and "arena_<r>" (unrelated texts first, so T's label starts at residue r)."""
    if shape == "one_node":
        return [(T, "http://w0")]
    if shape.startswith("split_"):
        k = int(shape.split("_")[1])
        return [(T, "http://w0"), (TB[:k].decode() + "Ω", "http://w1")]
    r = int(shape.split("_")[1])
    a = 7
    b = 16 + (r - a) % 16
    return [("#" + "x" * (a - 1), "http://w2"), ("%" + "y" * (b - 1), "http://w3"), (T, "http://w0")]


TEXT_SHAPES = ["one_node"] + [f"split_{k}" for k in SPLITS] + [f"arena_{r}" for r in ARENA_RESIDUES]


# =====================================================================================================================
# deep token conversations: request k = request k − 1 plus 1–3 new pages
# =====================================================================================================================
DEEP_DEPTHS = [31, 32, 33, 34, 64, 300]


def deep_conversations(seed=5):
    """one conversation per depth D: turns 0..D, each a fresh first page and 1–3 fresh pages per turn (ids disjoint across convs)"""
    rng = np.random.default_rng(seed)
    convs = []
    for c, d in enumerate(DEEP_DEPTHS):
        base = 200000 + c * 100000
        turns, cur, nxt = [], np.zeros(0, np.uint32), base
        for _ in range(d + 1):
            k = int(rng.integers(1, 4)) * PAGE
            cur = np.concatenate([cur, np.arange(nxt, nxt + k, dtype=np.uint32)])
            nxt += k
            turns.append(cur)
        convs.append(turns)
    return convs


def deep_schedule(convs, seed=6):
    """Batches of (conv, turn) items (turn −1 = a fresh shallow request).  Phase A: turn k of every conversation in batch k (first
    pages distinct); phase B: up to 8 consecutive turns of the two deepest conversations per batch (they share a first page), mixed with
    re-sends of turns inserted in earlier batches and shallow requests."""
    rng = np.random.default_rng(seed)
    batches, done = [], [0] * len(convs)
    for k in range(36):
        b = [(c, k) for c in range(len(convs)) if k < len(convs[c])]
        b += [(-1, int(rng.integers(1, 4)))] * 2
        batches.append(b)
        for c in range(len(convs)):
            done[c] = min(k + 1, len(convs[c]))
    while any(done[c] < len(convs[c]) for c in (4, 5)):
        b = []
        for c in (4, 5):
            m = min(8, len(convs[c]) - done[c])
            b += [(c, done[c] + j) for j in range(m)]
        for _ in range(3):
            c = int(rng.integers(0, len(convs)))
            b.insert(int(rng.integers(0, len(b) + 1)), (c, int(rng.integers(0, done[c]))))
        b.insert(int(rng.integers(0, len(b) + 1)), (-1, int(rng.integers(1, 4))))
        for c in (4, 5):
            done[c] = min(done[c] + 8, len(convs[c]))
        batches.append(b)
    return batches


def _request_of(convs, item, counter):
    c, k = item
    if c < 0:
        counter[0] += 1
        return np.arange(900000 + 64 * counter[0], 900000 + 64 * counter[0] + k * PAGE, dtype=np.uint32)
    return convs[c][k]


# =====================================================================================================================
# long chat stream (string tree, policy)
# =====================================================================================================================
def chat_stream(seed):
    """12 batches of routing texts: system prompts of 2–24 KB in mixed scripts, multi-turn conversations that each add a node per
    turn, repeats and cut prefixes."""
    r = random.Random(seed)
    prompts = [mixed_text(seed * 100 + i, r.randrange(2048, 24 * 1024)) for i in range(5)]
    convs = [[prompts[r.randrange(5)]] for _ in range(10)]
    batches = []
    for bno in range(12):
        texts = []
        for c in r.sample(range(10), 6):
            for _ in range(r.randrange(1, 4)):      # several turns of one conversation in one batch
                convs[c].append(convs[c][-1] + f"\nUser {len(convs[c])}: " + mixed_text(r.randrange(10 ** 6), r.randrange(20, 400)))
                texts.append(convs[c][-1])
        texts += [r.choice(prompts) + mixed_text(r.randrange(10 ** 6), r.randrange(1, 64)) for _ in range(3)]
        t = r.choice(texts)
        texts += [t, t[: r.randrange(len(t) + 1)], "", "你", r.choice(prompts)]
        r.shuffle(texts)
        batches.append(texts)
    return batches


# =====================================================================================================================
# request-start alignment
# =====================================================================================================================
def aligned_token_batch(longs, unit=4):
    """[short, long, short, long, ...] with shorts of 0..unit−1 tokens, so that long i starts at token offset ≡ i (mod unit)"""
    reqs, off, starts = [], 0, []
    for i, q in enumerate(longs):
        s = (i % unit - off) % unit
        reqs.append(np.arange(70000, 70000 + s, dtype=np.uint32))
        off += s
        starts.append(off)
        reqs.append(q)
        off += len(q)
    return reqs, starts


def aligned_text_batch(longs, unit=16):
    texts, off, starts = [], 0, []
    for i, q in enumerate(longs):
        s = (i % unit - off) % unit
        texts.append("z" * s)
        off += s
        starts.append(off)
        texts.append(q)
        off += len(q.encode())
    return texts, starts


ALIGN_TOKEN_LONGS = [c[1] for c in TOKEN_CASES if c[0].startswith(("mismatch", "ragged", "extend"))][:24]
ALIGN_TEXT_LONGS = ([c[1] for c in TEXT_CASES if c[2] in ("last", "lead", "extend")] * 3)[:32]


# =====================================================================================================================
# CPU: generators and the oracle against the closed forms
# =====================================================================================================================
def test_token_cases_sit_on_their_boundaries():
    assert len(S) == 1536 and S.max() < 50000
    seen = set()
    for name, q, kind, at in TOKEN_CASES:
        if kind == "mismatch":
            assert _lcp(q, S) == at and q[at] != S[at], name
            where = name.split("_")[1].split("@")[0] if name.startswith("mismatch_") else None
            if where:
                assert _on_boundary(where, at), name
            seen.add(at % 4)
        elif kind == "stop":
            assert len(q) == at and np.array_equal(q, S[:at]), name
        elif kind == "extend":
            assert np.array_equal(q[: len(S)], S) and len(q) > len(S) and len(q) % PAGE == 0, name
        else:
            assert np.array_equal(q[: len(S)], S) and len(q) % PAGE == at, name
    assert seen == {0, 1, 2, 3}
    # the split at page 5 really starts a label at token 80, which is not aligned to a round or a window
    assert _lcp(token_inserts("split_at_page_5")[1][0], S) == 80
    for p in TOKEN_SHAPES["chain"]:
        assert np.array_equal(token_inserts("chain")[1 + TOKEN_SHAPES["chain"].index(p)][0][: 16 * p], S[: 16 * p])


def test_text_cases_sit_on_their_boundaries():
    assert 12 * 1024 <= len(TB) < 12 * 1024 + 4
    for s in (2, 3, 4):
        assert sum(1 for ch in T if len(ch.encode()) == s) > 100        # really mixed
    for name, (b, c) in STRADDLES.items():
        n = len(c.encode())
        assert TB[b:b + n] == c.encode()
        for edge in STRADDLE_BOUNDARIES[name]:
            assert b < edge < b + n, name                               # the char covers bytes edge − 1 and edge
    for name, q, kind, at in TEXT_CASES:
        qb = q.encode()
        if kind in ("last", "lead"):
            b, c = STRADDLES[name.split("_byte_")[1]]
            n = len(c.encode())
            assert len(q) == len(T) and len(qb) == len(TB)
            first_diff = _lcp(np.frombuffer(qb, np.uint8), np.frombuffer(TB, np.uint8))
            assert first_diff == (b + n - 1 if kind == "last" else b), name
            if kind == "last":                                           # the mismatch byte lies past the boundary
                assert all(first_diff >= e for e in STRADDLE_BOUNDARIES[name.split("_byte_")[1]]), name
            assert len(os.path.commonprefix([q, T])) == _char_at(b), name
        elif kind == "end":
            assert qb == TB[:at]
        elif kind == "extend":
            assert qb[: len(TB)] == TB and len(qb) > len(TB)
    for k in SPLITS:
        assert k % 16 and TB[k] & 0xC0 != 0x80
    assert TB[4078] == 0xF0                                              # a 4-byte char starts 2 bytes before the window end
    for r in ARENA_RESIDUES:
        before = text_shape_inserts(f"arena_{r}")[:-1]
        assert sum(len(t.encode()) for t, _ in before) % 16 == r
        assert all(t[0] != T[0] for t, _ in before) and before[0][0][0] != before[1][0][0]


@pytest.mark.parametrize("shape", list(TOKEN_SHAPES))
def test_token_oracle_equals_closed_form(shape):
    orc.reset_globals()
    o = orc.TokenTree()
    ins = token_inserts(shape)
    for s, t in ins:
        o.insert_tokens(s, t)
    for name, q, _, _ in TOKEN_CASES:
        m = o.match_prefix_with_counts(q)
        assert m.matched_token_count == token_closed_form([s for s, _ in ins], q), name
        assert m.input_token_count == len(q)


@pytest.mark.parametrize("shape", TEXT_SHAPES)
def test_text_oracle_equals_closed_form(shape):
    orc.reset_globals()
    o = orc.Tree()
    ins = text_shape_inserts(shape)
    for s, t in ins:
        o.insert_text(s, t)
    for name, q, _, _ in TEXT_CASES:
        m = o.match_prefix_with_counts(q)
        assert m.matched_char_count == text_closed_form([s for s, _ in ins], q), name
        assert m.input_char_count == len(q)


def test_deep_conversations_have_the_depths_they_name():
    convs = deep_conversations()
    for d, turns in zip(DEEP_DEPTHS, convs):
        assert len(turns) == d + 1
        for a, b in zip(turns, turns[1:]):
            assert np.array_equal(b[: len(a)], a) and (len(b) - len(a)) // PAGE in (1, 2, 3) and len(b) % PAGE == 0
        orc.reset_globals()
        o = orc.TokenTree()
        for t in turns[:-1]:
            o.insert_tokens(t, "http://w0")
        m = o.match_prefix_with_counts(turns[-1])
        assert m.nodes_visited == d and m.matched_token_count == len(turns[-2])
    assert max(len(t[-1]) for t in convs) * 4 > 1024                    # hashes span several BLAKE3 chunks
    sched = deep_schedule(convs)
    assert any(sum(1 for c, _ in b if c == 5) > 1 for b in sched)       # deep requests sharing a first page in one batch
    assert all(any(c < 0 for c, _ in b) for b in sched)                 # every batch mixes in shallow requests
    nxt = {}
    for b in sched:                                                      # turns arrive in order; re-sends only of earlier batches
        before = dict(nxt)
        for c, k in b:
            if c < 0 or k < before.get(c, 0):
                continue
            assert k == nxt.get(c, 0)
            nxt[c] = k + 1
    assert [nxt[c] for c in range(len(convs))] == [d + 1 for d in DEEP_DEPTHS]


def test_alignment_batches_cover_every_residue():
    _, starts = aligned_token_batch(ALIGN_TOKEN_LONGS)
    assert {s % 4 for s in starts} == {0, 1, 2, 3}
    _, starts = aligned_text_batch(ALIGN_TEXT_LONGS)
    assert {s % 16 for s in starts} == set(range(16))


@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
def test_oracle_policy_sweep_equals_closed_form(mode):
    """The policy-level oracle on the token sweep (chain shape) and the text sweep (one node) agrees with the closed forms."""
    orc.reset_globals()
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **CFG)
    urls = synth.worker_urls(8)
    op.set_workers(urls)
    op.set_state([0] * 8, [1] * 8, [1] * 8)
    inserted = []
    for s, _ in token_inserts("chain"):
        d = op.select_worker(tokens=s)
        assert d.matched == token_closed_form(inserted, s)
        inserted.append(s)
    qs = [c[1] for c in TOKEN_CASES]
    if mode == "snapshot":
        flat, off = _flat(qs)
        _, br, ma, _ = op.select_batch_tokens(flat, off, snapshot=True)
        assert [int(x) for x in ma] == [token_closed_form(inserted, q) for q in qs]
    else:
        for q in qs:
            d = op.select_worker(tokens=q)
            assert d.matched == token_closed_form(inserted, q)
            if orc.BRANCHES.index(d.branch) in INSERTING:
                inserted.append(q)
    d = op.select_worker(request_text=T)
    texts = [c[1] for c in TEXT_CASES]
    if mode == "snapshot":
        _, _, ma, inp, _ = op.select_batch_text(texts, snapshot=True)
        assert [int(x) for x in ma] == [text_closed_form([T], q) for q in texts]
        assert [int(x) for x in inp] == [len(q) for q in texts]
    else:
        ins = [T]
        for q in texts:
            d = op.select_worker(request_text=q)
            assert d.matched == text_closed_form(ins, q) and d.input == len(q)
            if orc.BRANCHES.index(d.branch) in INSERTING:
                ins.append(q)


# =====================================================================================================================
# GPU helpers
# =====================================================================================================================
def _flat(reqs):
    flat = np.concatenate([np.asarray(r, np.uint32) for r in reqs]) if sum(len(r) for r in reqs) else np.zeros(0, np.uint32)
    off = np.zeros(len(reqs) + 1, np.uint64)
    np.cumsum([len(r) for r in reqs], out=off[1:])
    return flat, off


def _pair(n_workers, mode):
    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
    urls = synth.worker_urls(n_workers)
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **CFG), tree_batch_mode=mode)
    ws = [BasicWorker(u) for u in urls]
    pol.init_workers(ws)
    orc.reset_globals()
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **CFG)
    op.set_workers(urls)
    return pol, ws, op, urls


def _set_fleet(ws, op, loads, healthy):
    for w, l, h in zip(ws, loads, healthy):
        w.set_load(int(l)); w.set_healthy(bool(h))
    op.set_state(loads, healthy, [1] * len(ws))


def _route_tokens(pol, ws, op, reqs, mode, tag, inserted=None):
    """One batch through the GPU path and the oracle: pick, branch, matched and input per request (and the closed form while the
    tree has only seen inserts)."""
    idx, info = pol.select_worker_batch(ws, reqs)
    if mode == "snapshot":
        flat, off = _flat(reqs)
        want, br, ma, _ = op.select_batch_tokens(flat, off, snapshot=True)
        for i in range(len(reqs)):
            assert (want[i], br[i], ma[i], len(reqs[i])) == (idx[i], info[i].branch, info[i].matched, info[i].input), (tag, i)
        if inserted is not None:
            for i, r in enumerate(reqs):
                assert info[i].matched == token_closed_form(inserted, r), (tag, i)
            inserted += [r for i, r in enumerate(reqs) if info[i].branch in INSERTING and idx[i] >= 0]
    else:
        for i, r in enumerate(reqs):
            d = op.select_worker(tokens=r)
            assert (d.idx if d.idx is not None else -1) == idx[i], (tag, i, d.branch, orc.BRANCHES[info[i].branch])
            assert d.branch == orc.BRANCHES[info[i].branch] and d.matched == info[i].matched and d.input == info[i].input, (tag, i)
            if inserted is not None:
                assert info[i].matched == token_closed_form(inserted, r), (tag, i)
                if info[i].branch in INSERTING and idx[i] >= 0:
                    inserted.append(r)
    return idx, info


def _route_text(pol, ws, op, texts, mode, tag, inserted=None):
    idx, info = pol.select_worker_batch_request_text(ws, texts)
    if mode == "snapshot":
        want, br, ma, inp, _ = op.select_batch_text(texts, snapshot=True)
        for i in range(len(texts)):
            assert (want[i], br[i], ma[i], inp[i]) == (idx[i], info[i].branch, info[i].matched, info[i].input), (tag, i)
        if inserted is not None:
            for i, t in enumerate(texts):
                assert info[i].matched == text_closed_form(inserted, t), (tag, i)
            inserted += [t for i, t in enumerate(texts) if info[i].branch in INSERTING and idx[i] >= 0]
    else:
        for i, t in enumerate(texts):
            d = op.select_worker(request_text=t)
            assert (d.idx if d.idx is not None else -1) == idx[i], (tag, i, d.branch, orc.BRANCHES[info[i].branch])
            assert d.branch == orc.BRANCHES[info[i].branch] and d.matched == info[i].matched and d.input == info[i].input, (tag, i)
            if inserted is not None:
                assert info[i].matched == text_closed_form(inserted, t), (tag, i)
                if info[i].branch in INSERTING and idx[i] >= 0:
                    inserted.append(t)
    return idx, info


def _same_token_state(pol, op, urls, hashes=True):
    assert pol.token_tree().entries() == op.token_tree().entries()      # same nodes, tenants and timestamps
    for u in urls:
        assert pol.token_tree().tenant_token_size(u) == op.token_tree().tenant_token_size(u)
    if hashes:
        want = op.hash_index("tokens")
        assert pol.hash_index_size("tokens") == len(want)
        for h, prefix in want.items():
            assert pol.hash_index_get(h, "tokens") == prefix


def _same_text_state(pol, op):
    st, ot = pol.string_tree(), op.string_tree()
    assert st.entries() == ot.entries()
    assert st.get_tenant_char_count() == ot.get_tenant_char_count()
    assert st.get_used_size_per_tenant() == ot.get_used_size_per_tenant()
    assert st.node_count() == ot.node_count()
    want = op.hash_index("text")
    assert pol.hash_index_size("text") == len(want)
    for h, prefix in want.items():
        assert pol.hash_index_get(h, "text") == prefix


# =====================================================================================================================
# 1. token tree: mismatch sweep
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(TOKEN_SHAPES))
def test_token_sweep_standalone(shape):
    from smg_b200 import TokenTree
    t = TokenTree.standalone()
    orc.reset_globals()
    o = orc.TokenTree()
    ins = token_inserts(shape)
    for s, ten in ins:
        t.insert_tokens(s, ten)
        o.insert_tokens(s, ten)
    for name, q, _, _ in TOKEN_CASES:
        g, w = t.match_prefix_with_counts(q), o.match_prefix_with_counts(q)
        assert (g.matched_token_count, g.input_token_count, g.tenant) == (w.matched_token_count, w.input_token_count, w.tenant), name
        assert g.matched_token_count == token_closed_form([s for s, _ in ins], q), name
    assert t.entries() == o.entries()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
@pytest.mark.parametrize("shape", list(TOKEN_SHAPES))
def test_token_sweep_policy(shape, mode):
    pol, ws, op, urls = _pair(8, mode)
    _set_fleet(ws, op, [3, 0, 5, 1, 2, 7, 4, 6], [1] * 8)
    inserted = []
    ins = [s for s, _ in token_inserts(shape)]
    _route_tokens(pol, ws, op, ins[:1], mode, "base", inserted)
    if len(ins) > 1:
        _route_tokens(pol, ws, op, ins[1:], mode, "branches", inserted)
    _route_tokens(pol, ws, op, [c[1] for c in TOKEN_CASES], mode, "sweep", inserted)
    _same_token_state(pol, op, urls)


# =====================================================================================================================
# 2. token tree: deep chains
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
def test_deep_chains_policy(mode):
    pol, ws, op, urls = _pair(8, mode)
    convs = deep_conversations()
    rng = np.random.default_rng(9)
    counter = [0]
    turns_in = [0] * len(convs)            # turns of each conversation inserted so far
    for bno, batch in enumerate(deep_schedule(convs)):
        loads = rng.integers(0, 12, size=8)
        if bno == 20:
            loads[0] += 200                # imbalanced batch: min-load picks that still insert
        _set_fleet(ws, op, loads, [1] * 8)
        reqs = [_request_of(convs, it, counter) for it in batch]
        before = list(turns_in)
        idx, info = _route_tokens(pol, ws, op, reqs, mode, bno)
        for i, (c, k) in enumerate(batch):
            assert info[i].branch in INSERTING and idx[i] >= 0
            if c < 0:
                assert info[i].nodes == 0, (bno, i)
                continue
            if k < before[c]:              # a re-send of an inserted turn: its own node too
                want = k + 1
            else:
                want = k if mode == "sequential" else before[c]
                turns_in[c] = max(turns_in[c], k + 1)
            assert info[i].nodes == min(want, 255), (bno, i, c, k, info[i].nodes)
        _same_token_state(pol, op, urls, hashes=(bno % 10 == 0))
    assert turns_in == [d + 1 for d in DEEP_DEPTHS]
    _same_token_state(pol, op, urls)
    pol.evict_cache(3000)
    op.evict_cache(3000)
    _same_token_state(pol, op, urls)


# =====================================================================================================================
# 3. string tree: mismatch sweep with UTF-8 straddles
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("shape", TEXT_SHAPES)
def test_text_sweep_standalone(shape):
    from smg_b200.policy import Tree
    t = Tree.standalone()
    orc.reset_globals()
    o = orc.Tree()
    ins = text_shape_inserts(shape)
    for s, ten in ins:
        t.insert_text(s, ten)
        o.insert_text(s, ten)
    for name, q, _, _ in TEXT_CASES:
        g, w = t.match_prefix_with_counts(q), o.match_prefix_with_counts(q)
        assert (g.matched_char_count, g.input_char_count, g.tenant) == (w.matched_char_count, w.input_char_count, w.tenant), name
        assert g.matched_char_count == text_closed_form([s for s, _ in ins], q), name
    assert t.entries() == o.entries()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
@pytest.mark.parametrize("shape", ["one_node", "split_509", "split_4078", "arena_5"])
def test_text_sweep_policy(shape, mode):
    pol, ws, op, urls = _pair(8, mode)
    _set_fleet(ws, op, [3, 0, 5, 1, 2, 7, 4, 6], [1] * 8)
    inserted = []
    for s, _ in text_shape_inserts(shape):
        _route_text(pol, ws, op, [s], mode, "build", inserted)
    _route_text(pol, ws, op, [c[1] for c in TEXT_CASES], mode, "sweep", inserted)
    _same_text_state(pol, op)


# =====================================================================================================================
# 4. string tree: long chat stream
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
@pytest.mark.parametrize("seed,n_workers", [(1, 4), (2, 16)])
def test_long_chat_stream_parity(seed, n_workers, mode):
    pol, ws, op, urls = _pair(n_workers, mode)
    rng = np.random.default_rng(seed)
    for bno, texts in enumerate(chat_stream(seed)):
        loads = rng.integers(0, 12, size=n_workers)
        healthy = (rng.random(n_workers) > 0.1).astype(np.uint8)
        if bno == 7:
            loads[0] += 200
        _set_fleet(ws, op, loads, healthy)
        _route_text(pol, ws, op, texts, mode, bno)
        if bno == 5:
            pol.evict_cache(20000)
            op.evict_cache(20000)
            assert pol.string_tree().entries() == op.string_tree().entries()
    _same_text_state(pol, op)
    assert list(pol.take_processed()) == [op.processed(i) for i in range(n_workers)]


# =====================================================================================================================
# 5. request start alignment: batch calls and the device-resident walks
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
def test_token_request_start_alignment(mode):
    pol, ws, op, urls = _pair(8, mode)
    _set_fleet(ws, op, [3, 0, 5, 1, 2, 7, 4, 6], [1] * 8)
    inserted = []
    _route_tokens(pol, ws, op, [s for s, _ in token_inserts("chain")], mode, "build", inserted)
    reqs, _ = aligned_token_batch(ALIGN_TOKEN_LONGS)
    _route_tokens(pol, ws, op, reqs, mode, "aligned", inserted)
    _same_token_state(pol, op, urls)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
def test_text_request_start_alignment(mode):
    pol, ws, op, urls = _pair(8, mode)
    _set_fleet(ws, op, [3, 0, 5, 1, 2, 7, 4, 6], [1] * 8)
    inserted = []
    for s, _ in text_shape_inserts("split_509"):
        _route_text(pol, ws, op, [s], mode, "build", inserted)
    texts, _ = aligned_text_batch(ALIGN_TEXT_LONGS)
    _route_text(pol, ws, op, texts, mode, "aligned", inserted)
    _same_text_state(pol, op)


class _Dev:
    """device buffers of one policy handle, freed together"""

    def __init__(self, pol):
        from smg_b200 import _lib
        self.h, self.L, self.ptrs = pol._h, _lib.load(), []
        self.depth = self.L.smgx_pipeline_depth(self.h.p)

    def put(self, arr, shift=0):
        """copy arr to a fresh device buffer `shift` bytes past its (aligned) start; → device address of the copy"""
        from smg_b200 import _lib
        err = _lib.new_err()
        p = self.L.smgx_device_alloc(self.h.p, arr.nbytes + shift + 16, C.byref(err))
        assert p, err.value
        self.ptrs.append(p)
        if arr.nbytes:
            self.h.call("smgx_memcpy_h2d", C.c_void_p(p + shift), arr.ctypes.data_as(C.c_void_p), arr.nbytes)
        return p + shift

    def get(self, dptr, arr):
        self.h.call("smgx_memcpy_d2h", arr.ctypes.data_as(C.c_void_p), C.c_void_p(dptr), arr.nbytes)
        return arr

    def free(self):
        for p in self.ptrs:
            self.L.smgx_device_free(self.h.p, p)
        self.ptrs = []


def _ptrs(xs):
    return (C.c_void_p * len(xs))(*xs)


@pytest.mark.gpu
def test_token_walk_many_device():
    """smgx_tree_walk_many_device: batches at device addresses offset by 0–3 tokens, more batches than stream lanes; the walk is
    read-only, so all batches together equal one oracle snapshot call on the same tree."""
    from smg_b200 import _lib
    pol, ws, op, urls = _pair(8, "sequential")
    _set_fleet(ws, op, [3, 0, 5, 1, 2, 7, 4, 6], [1] * 8)
    _route_tokens(pol, ws, op, [s for s, _ in token_inserts("chain")], "sequential", "build")
    convs = deep_conversations()
    for k in range(36):                    # a 36-deep chain: walks past kPathCap
        _route_tokens(pol, ws, op, [convs[4][k]], "sequential", k)
    model = pol._push_fleet(ws)
    entries = pol.token_tree().entries()
    dev = _Dev(pol)
    try:
        nb = 2 * dev.depth + 1
        queries = [c[1] for c in TOKEN_CASES] + [convs[4][35], convs[4][36], convs[4][10]]
        batches = [queries[j::nb] for j in range(nb)]
        d_tok, d_off, d_out, d_info, ns = [], [], [], [], []
        for j, b in enumerate(batches):
            flat, off = _flat(b)
            d_tok.append(dev.put(flat, 4 * (j % 4)))
            d_off.append(dev.put(off.astype(np.uint32)))
            d_out.append(dev.put(np.full(len(b), -7, np.int32)))
            d_info.append(dev.put(np.zeros(len(b) * C.sizeof(_lib.DecisionInfo), np.uint8)))
            ns.append(len(b))
        pol._h.call("smgx_tree_walk_many_device", model, nb, _ptrs(d_tok), _ptrs(d_off), (C.c_uint32 * nb)(*ns), _ptrs(d_out), _ptrs(d_info))
        pol._h.call("smgx_synchronize")
        got_idx, got_info = [], []
        for j in range(nb):
            got_idx += list(dev.get(d_out[j], np.zeros(ns[j], np.int32)))
            info = (_lib.DecisionInfo * ns[j])()
            pol._h.call("smgx_memcpy_d2h", C.cast(info, C.c_void_p), C.c_void_p(d_info[j]), C.sizeof(info))
            got_info += list(info)
    finally:
        dev.free()
    assert pol.token_tree().entries() == entries                         # read-only
    allq = [q for b in batches for q in b]
    flat, off = _flat(allq)
    want, br, ma, _ = op.select_batch_tokens(flat, off, snapshot=True)
    for i, q in enumerate(allq):
        assert (want[i], br[i], ma[i], len(q)) == (got_idx[i], got_info[i].branch, got_info[i].matched, got_info[i].input), i


@pytest.mark.gpu
def test_text_walk_many_device():
    """smgx_stree_walk_many_device: text batches at device addresses offset by 0–15 bytes, more batches than stream lanes."""
    from smg_b200 import _lib
    pol, ws, op, urls = _pair(8, "sequential")
    _set_fleet(ws, op, [3, 0, 5, 1, 2, 7, 4, 6], [1] * 8)
    for s, _ in text_shape_inserts("split_4078"):
        _route_text(pol, ws, op, [s], "sequential", "build")
    model = pol._push_fleet(ws)
    entries = pol.string_tree().entries()
    dev = _Dev(pol)
    try:
        nb = max(2 * dev.depth + 1, 16)
        queries = [c[1] for c in TEXT_CASES]
        batches = [queries[j::nb] for j in range(nb)]
        d_txt, d_off, d_out, d_info, d_node, ns = [], [], [], [], [], []
        for j, b in enumerate(batches):
            enc = [t.encode() for t in b]
            data = np.frombuffer(b"".join(enc) or b"\0", np.uint8).copy()
            off = np.zeros(len(b) + 1, np.uint32)
            np.cumsum([len(e) for e in enc], out=off[1:])
            d_txt.append(dev.put(data, j % 16))
            d_off.append(dev.put(off))
            d_out.append(dev.put(np.full(max(len(b), 1), -7, np.int32)))
            d_info.append(dev.put(np.zeros(max(len(b), 1) * C.sizeof(_lib.DecisionInfo), np.uint8)))
            d_node.append(dev.put(np.zeros(max(len(b), 1), np.uint32)))
            ns.append(len(b))
        pol._h.call("smgx_stree_walk_many_device", model, nb, _ptrs(d_txt), _ptrs(d_off), (C.c_uint32 * nb)(*ns), _ptrs(d_out), _ptrs(d_info),
                    _ptrs(d_node))
        pol._h.call("smgx_synchronize")
        got_idx, got_info = [], []
        for j in range(nb):
            if not ns[j]:
                continue
            got_idx += list(dev.get(d_out[j], np.zeros(ns[j], np.int32)))
            info = (_lib.DecisionInfo * ns[j])()
            pol._h.call("smgx_memcpy_d2h", C.cast(info, C.c_void_p), C.c_void_p(d_info[j]), C.sizeof(info))
            got_info += list(info)
    finally:
        dev.free()
    assert pol.string_tree().entries() == entries
    allq = [q for b in batches for q in b]
    want, br, ma, inp, _ = op.select_batch_text(allq, snapshot=True)
    for i, q in enumerate(allq):
        assert (want[i], br[i], ma[i], inp[i]) == (got_idx[i], got_info[i].branch, got_info[i].matched, got_info[i].input), i
        assert got_info[i].matched == text_closed_form([T, TB[:4078].decode() + "Ω"], q), i
