"""Pipelined submissions against the oracle while the index, the fleet and the routing mode change between submissions.

The gateway reaches the GPU through the pipelined calls (smgx_submit_tokens / smgx_wait, smgx_submit_text, smgx_submit_tokens_mapped,
smgx_select_batch_tokens_device on explicit lanes, smgx_select_many_tokens_device).  Each of the policy's lanes has its own stream and
staging, so up to smgx_pipeline_depth() batches are in flight while the host keeps applying KV events, fleet snapshots and worker
changes.  Every submission must be decided against the state at the moment it was submitted: sync_state makes the ctrl stream wait for
every lane's `done` event before EventIndex::flush updates the device copy, and smgx_wait synchronises the lane before it returns.

build_plan() makes a seeded sequence of submissions and state transitions; run_oracle() replays it on the oracle, each submission
against exactly the transitions that precede it.  Every transition sits between two submissions that are both in flight, and each
reaches one path of flush / sync_state: the scatter (slots, tags, run records, a Multi entry at position 1, bitset rows with more than
64 workers), the full re-upload (more than 1/8 of the slots dirty), the rebuild (the table crosses half load), the bitset width growth
(the 65th worker), a run compaction, apply_cleared / remove_worker, new loads and health, larger and duplicate worker slices, and an
imbalanced fleet and back.  The CPU test checks the plan for all of that; the GPU tests run it with every transport.

Before each submission the lane it takes is held by a ~2 ms hold kernel, so the submission is really still queued when the host
applies the next transition.  Outputs are poisoned; with pinned output buffers the copy back is truly asynchronous, so a wait that
returned before its lane finished shows up as poison."""
import ctypes as C
import functools
import os
import time

import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth
from tests import consistent_hashing_oracle as ch
from tests.test_gpu_event_sequences import (BS, IMBALANCED, INFO, INFO_POISON, MAX_BLOCKS, MIN_LOAD, NO_HEALTHY, OVERLAP, POISON, Device,
                                            apply_ops, check, gpu_policy, oracle_policy, poisoned_info, ragged, set_fleet)

W0, W_ALL = 64, 70          # workers interned at the start / after the width growth
MAX_TOKENS = 8 * MAX_BLOCKS * BS   # max_tokens_per_request: text submissions bound a request by its bytes
HOLD_US = 2000
TOKEN_POISON = 0xA5A5A5A5
VOCAB_FILE = os.path.join(os.path.dirname(__file__), "golden", "synth_vocab.tiktoken")
SMGX_BUSY, SMGX_INVALID_ARGUMENT, SMGX_NOT_FOUND = 13, 1, 12
TREE_MATCH, TREE_MIN_LOAD = 4, 5

# the transitions a plan must place between two in-flight submissions (see the module docstring)
INITIAL_FLEET = (np.full(W0, 5, np.uint64), np.ones(W0, np.uint8), np.ones(W0, np.uint8))
TRANSITIONS = ["scatter", "full", "grow", "intern65", "rows", "compact", "cleared", "fleet", "slice_grow", "slice_dup", "imbalanced",
               "balanced", "no_healthy"]


# ---- the plan (pure data, no GPU) -------------------------------------------------------------------------------------------------

class IndexModel:
    """What EventIndex's host side does with the plan's ops, as far as the upload path of the next flush depends on it: live keys
    (position, content hash), tombstones (an upper bound: a new key may re-use one on its probe path), the slot capacity (a lower bound
    once a rebuild may have happened early because of tombstones), the bitset width and the run records appended."""

    def __init__(self):
        self.cap, self.words, self.n_workers = 1024, 1, 0
        self.holders = {}   # (pos, content) → {(prefix, worker)}
        self.blocks = {}    # (worker, seq hash) → (pos, content, prefix)
        self.tombs = 0
        self.records = 0    # run records appended so far
        self.max_live = 0
        self.begin()

    def begin(self):
        self.t = dict(touched=0, new_keys=0, killed=0, reborn=0, multi1=False, widened=False, dead_records=0, records_before=self.records,
                      live_before=self.live(), tombs_before=self.tombs, cap_before=self.cap, words_before=self.words, grew=False)
        self.dead_keys = set()

    def live(self):
        return len(self.holders)

    def intern(self):
        wid = self.n_workers
        self.n_workers += 1
        if wid >= self.words * 64:
            self.words *= 2
            self.tombs = 0
            self.t["widened"] = True
        return wid

    def store(self, w, blocks):
        prefix = 0
        for pos, (seq, c) in enumerate(blocks):
            prefix = hash((prefix, c)) if pos else c
            key = (pos, c)
            self.records += 1
            self.t["touched"] += 1
            hs = self.holders.get(key)
            if hs is None:
                if key in self.dead_keys:
                    self.t["reborn"] += 1
                self.holders[key] = {(prefix, w)}
                self.t["new_keys"] += 1
                if (self.live() + 1) * 2 > self.cap:   # a rebuild for certain (tombstones can only bring it earlier)
                    while (self.live() + 1) * 4 > self.cap:
                        self.cap *= 2
                    self.tombs = 0
                    self.t["grew"] = True
            else:
                self.t["dead_records"] += 1
                if pos == 1 and all(p != prefix for p, _ in hs):
                    self.t["multi1"] = True
                hs.add((prefix, w))
            self.blocks[(w, seq)] = (pos, c, prefix)
        self.max_live = max(self.max_live, self.live())

    def remove(self, w, seqs):
        for s in seqs:
            rec = self.blocks.pop((w, s), None)
            if rec is None:
                continue
            pos, c, prefix = rec
            self.t["touched"] += 1
            hs = self.holders[(pos, c)]
            hs.discard((prefix, w))
            if not hs:
                del self.holders[(pos, c)]
                self.tombs += 1
                self.t["killed"] += 1
                self.dead_keys.add((pos, c))

    def clear(self, w):
        self.remove(w, [s for (ww, s) in list(self.blocks) if ww == w])


def _fleet(rng, n, kind):
    loads = rng.integers(0, 21, size=n).astype(np.uint64)
    healthy, circuit = np.ones(n, np.uint8), np.ones(n, np.uint8)
    if kind == "imbalanced":
        loads[int(rng.integers(0, n))] = 400
    elif kind == "one_down":
        down, tripped = rng.choice(n, size=2, replace=False)
        healthy[down] = 0
        circuit[tripped] = 0
    elif kind == "none":
        healthy[:] = 0
    return loads, healthy, circuit


# requests per submission: lane staging grows (40 → 120 → 200) and shrinks again, empty submissions included
SIZES = [6, 40, 3, 120, 0, 17, 64, 9, 200, 2, 33, 80, 1, 150, 12, 5, 90, 24, 0, 48, 7, 130, 20, 4, 60, 11, 3]
KINDS = ["hit", "partial", "novel", "long", "tiny", "empty", "multi", "hit", "partial", "long"]


@functools.lru_cache(maxsize=None)
def build_plan(jump, text_seed=None):
    """→ dict(urls, init (index ops), steps).  A step is ("submit", reqs, pad, kinds) or ("T", name, ops): ops are
    ("stored", w, blocks), ("removed", w, seqs), ("cleared", w, None), ("remove_worker", w, None), ("intern", url, None),
    ("slice", urls, None) and ("fleet", (loads, healthy, circuit), None).  With text_seed the token sequences come from ASCII texts
    encoded by the synthetic cl100k-shaped vocabulary (needs tiktoken), so that every request decodes to valid text."""
    rng = np.random.default_rng(7000 + jump + (text_seed or 0))
    urls = synth.worker_urls(W_ALL)
    L = MAX_BLOCKS * BS
    if text_seed is None:
        pool = [np.asarray(s, np.uint32) for s in synth.gen_sequences(40, L, 500 + jump)]

        def noise(n):
            return rng.integers(0, synth.VOCAB, size=n, dtype=np.uint32)
    else:
        enc = text_encoding()
        pool = [np.asarray(enc.encode(ascii_text(rng, 6 * L)), np.uint32)[:L] for _ in range(40)]
        assert all(p.size == L for p in pool)

        def noise(n):
            return np.asarray(enc.encode(ascii_text(rng, 4 * n + 8)), np.uint32)[:n]
    model = IndexModel()
    sid = [1]
    depth_of, held = {}, {}    # sequence → stored depth; worker → [(sequence, seq hashes)]

    def store(w, tokens, depth, s=None, keep=True):
        hs = orc.compute_request_content_hashes(tokens[:depth * BS], BS)
        blocks = [(sid[0] + i, hs[i]) for i in range(depth)]
        sid[0] += depth
        model.store(w, blocks)
        if keep:
            held.setdefault(w, []).append((s, [b[0] for b in blocks]))
        if s is not None:
            depth_of[s] = max(depth_of.get(s, 0), depth)
        return ("stored", w, blocks)

    def remove(w, seqs):
        model.remove(w, seqs)
        return ("removed", w, seqs)

    init = []
    for _ in range(W0):
        model.intern()
    for s in range(20):   # about 280 live keys: the table stays at 1024 slots until "grow"
        d = 40 if s < 4 else int(rng.integers(3, 13))
        for w in rng.choice(W0, size=int(rng.integers(1, 3)), replace=False):
            init.append(store(int(w), pool[s], d, s))
    # Multi entries at position 1: the same block 1 under two prefixes; m1 is stored at the start, its twin by "scatter"
    m0, m1, x0, x1 = (pool[36].copy(), pool[37].copy(), pool[38].copy(), pool[39].copy())
    x0[BS:2 * BS] = m0[BS:2 * BS]
    x1[BS:2 * BS] = m1[BS:2 * BS]
    init += [store(1, m0, 4, keep=False), store(2, x0, 2, keep=False), store(3, m1, 4, keep=False)]
    multi = [m0[:4 * BS], x0[:2 * BS], m1[:4 * BS], x1[:2 * BS]]
    next_seq = 20
    slice_urls = tuple(urls[:W0])

    def request(kind):
        s = int(rng.integers(0, next_seq))
        if kind == "empty":
            return np.zeros(0, np.uint32)
        if kind == "tiny":
            return pool[s][:int(rng.integers(1, BS))].copy()
        if kind == "multi":
            return multi[int(rng.integers(0, 4))].copy()
        if kind == "novel":
            return noise(int(rng.integers(1, MAX_BLOCKS + 1)) * BS)
        if kind == "long":   # more than 32 blocks: the slow kernel
            s = int(rng.integers(0, 4))
            return pool[s][:int(rng.integers(33, MAX_BLOCKS + 1)) * BS].copy()
        d = depth_of.get(s, 1)
        if kind == "hit":
            r = pool[s][:d * BS].copy()
        else:   # a cached prefix with a novel tail
            k = int(rng.integers(1, d + 1))
            r = np.concatenate([pool[s][:k * BS], noise(int(rng.integers(1, 12)) * BS)])
        if rng.random() < 0.3:
            r = np.concatenate([r, noise(int(rng.integers(1, BS)))])
        return r

    def fleet(kind, n=None):
        return ("fleet", _fleet(rng, n or len(slice_urls), kind), None)

    steps = []
    sizes = iter(SIZES)

    def submit():
        n = next(sizes)
        kinds = [KINDS[int(rng.integers(0, len(KINDS)))] for _ in range(n)]
        steps.append(("submit", [request(k) for k in kinds], int(rng.integers(0, 6)), kinds))

    def transition(name, ops):
        steps.append(("T", name, ops))
        model.begin()

    model.begin()
    submit(); submit()
    # scatter: a Multi at position 1, a tail evicted, the same blocks re-stored (onto the tombstones) by another worker, a new sequence
    ops = [store(4, x1, 2, keep=False)]
    holders_of = {}
    for w, lst in held.items():
        for s_, sq in lst:
            holders_of.setdefault(s_, []).append((w, sq))
    s = next(s_ for s_ in sorted(holders_of) if s_ >= 4 and len(holders_of[s_]) == 1 and depth_of[s_] >= 4)
    w_s, seqs = holders_of[s][0]
    ops.append(remove(w_s, seqs[-3:]))
    ops.append(store((w_s + 1) % W0, pool[s], depth_of[s]))
    ops.append(store(9, pool[next_seq], 3, next_seq)); next_seq += 1
    transition("scatter", ops)
    submit()
    transition("fleet", [fleet("one_down")]); submit()
    transition("imbalanced", [fleet("imbalanced")]); submit()
    transition("balanced", [fleet("balanced")]); submit()
    # full re-upload: evict more than 1/8 of the slots, without growth
    ops = []
    for w in sorted(held):
        keep = []
        for s_, seqs_ in held[w]:
            if s_ is not None and s_ >= 4 and len(ops) < 40:
                ops.append(remove(w, seqs_))
                depth_of[s_] = 1
            else:
                keep.append((s_, seqs_))
        held[w] = keep
    transition("full", ops); submit()
    transition("no_healthy", [fleet("none")]); submit()
    transition("balanced", [fleet("balanced")]); submit()
    # growth: new sequences until more than half of the 1024 slots are live
    ops = []
    while model.live() * 2 <= 1024 + 64:
        ops.append(store(int(rng.integers(0, W0)), pool[next_seq], MAX_BLOCKS, next_seq))
        next_seq += 1
    transition("grow", ops); submit()
    # the 65th worker: bitset width 1 → 2, rows, a new workers_version; the newcomers store existing and new blocks
    ops = [("intern", u, None) for u in urls[W0:]]
    for _ in urls[W0:]:
        model.intern()
    ops += [store(W0, pool[0], 40, 0), store(W0 + 1, pool[1], 20, 1), store(W0 + 2, pool[next_seq], 8, next_seq)]
    next_seq += 1
    transition("intern65", ops); submit()
    # row scatter: existing keys gain and lose workers of the second bitset word
    ops = [store(W0 + 3, pool[2], 12, 2), store(W0 + 4, pool[3], 6, 3), remove(W0, held[W0][0][1][-4:])]
    transition("rows", ops); submit()
    slice_urls = tuple(urls)
    transition("slice_grow", [("slice", slice_urls, None), fleet("balanced")]); submit()
    # run compaction: a worker adds itself to an existing run and leaves again until dead records outnumber the live entries
    ops = []
    budget = 2 * model.records + 2 * model.max_live + 1024 + 2 * MAX_BLOCKS
    owners = {w for w, lst in held.items() if any(s_ == 0 for s_, _ in lst)}   # a churn worker must not hold the run itself
    churn = [w for w in range(W_ALL) if w not in owners]
    while model.t["dead_records"] <= budget:
        w = churn[int(rng.integers(0, len(churn)))]
        op_ = store(w, pool[0], 40, keep=False)
        ops += [op_, remove(w, [b[0] for b in op_[2]])]
    transition("compact", ops); submit()
    transition("cleared", [("cleared", 7, None), ("remove_worker", 8, None)])
    model.clear(7); model.clear(8)
    submit()
    transition("imbalanced", [fleet("imbalanced")]); submit()
    slice_urls = tuple(urls) + (urls[5],)
    transition("slice_dup", [("slice", slice_urls, None), fleet("balanced")]); submit()
    transition("fleet", [fleet("one_down")]); submit()
    submit()
    return dict(urls=urls, jump=jump, init=init, steps=steps)


def ascii_text(rng, n):
    words = ["the", "route", "worker", "cache", "token", "prefix", "kernel", "lane", "batch", "alpha", "beta", "gamma", "x", "Q7", "zz"]
    out, size = [], 0
    while size < n:
        w = words[int(rng.integers(0, len(words)))] + (", " if rng.random() < 0.1 else " ")
        out.append(w)
        size += len(w)
    return "".join(out)


@functools.lru_cache(maxsize=None)
def text_encoding():
    """Live tiktoken over the synthetic cl100k-shaped vocabulary (the reference tokens of text requests)."""
    tiktoken = pytest.importorskip("tiktoken")
    import json
    from oracle import bpe_ref
    g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bpe_vectors.json")))
    return tiktoken.Encoding("synth", pat_str=g["pattern"], mergeable_ranks=bpe_ref.load_tiktoken_bpe(VOCAB_FILE), special_tokens=g["specials"])


def plan_texts(plan):
    """The text form of every submission's requests and their reference tokens (live tiktoken on that text)."""
    enc = text_encoding()
    out = []
    for st in plan["steps"]:
        if st[0] != "submit":
            out.append(None)
            continue
        texts = [enc.decode_bytes(r.tolist()).decode("ascii") for r in st[1]]
        out.append((texts, [np.asarray(enc.encode(t, allowed_special="all"), np.uint32) for t in texts]))
    return out


def apply_plan_ops(target, ops, gpu):
    """Index, slice and fleet changes, on the GPU run (gpu=True: target = Run) or the oracle (target = (policy, indexer, state))."""
    for op, a, b in ops:
        if op in ("stored", "removed"):
            apply_ops(target.ix if gpu else target[1], [(op, a, b)])
        elif op == "cleared":
            (target.ix if gpu else target[1]).apply_cleared(a)
        elif op == "remove_worker":
            (target.ix if gpu else target[1]).remove_worker(a)
        elif op == "intern":
            (target.ix if gpu else target[1]).intern_worker(a)
        elif op == "slice":
            if gpu:
                target.set_slice(a)
            else:
                target[0].set_workers(list(a))
        elif op == "fleet":
            if gpu:
                target.push_fleet(a)
            else:
                target[0].set_state(*a)


@functools.lru_cache(maxsize=None)
def run_oracle(jump, text_seed=None):
    """Per submission (in plan order): (picks, branches, matched tokens, request lengths); and the oracle's processed counters at the
    end, over the final slice."""
    plan = build_plan(jump, text_seed)
    texts = plan_texts(plan) if text_seed is not None else None
    op, oix = oracle_policy(plan["urls"][:W0], jump)
    apply_ops(oix, plan["init"])
    op.set_state(*INITIAL_FLEET)
    out = []
    n_slice = W0
    for k, st in enumerate(plan["steps"]):
        if st[0] == "T":
            apply_plan_ops((op, oix), st[2], gpu=False)
            n_slice = next((len(a) for o, a, _ in st[2] if o == "slice"), n_slice)
            continue
        reqs = texts[k][1] if texts else st[1]
        tokens, offsets, lens = ragged(reqs)
        if reqs:
            idx, br, ma, _ = op.select_batch_tokens(tokens, offsets.astype(np.uint64))
        else:
            idx, br, ma = np.zeros(0, np.int32), np.zeros(0, np.uint8), np.zeros(0, np.uint32)
        out.append((k, (np.asarray(idx), np.asarray(br), np.asarray(ma)), lens))
    return out, np.array([op.processed(i) for i in range(n_slice)], np.uint64)


@pytest.mark.parametrize("jump", [64, 8])
def test_plan_puts_every_transition_between_in_flight_submissions(jump):
    """CPU guard of the GPU tests: every transition sits between two submissions (the GPU runs never wait for the submission just
    before a transition until the one after it is submitted), each reaches the flush path it is named after by the documented
    thresholds (1/8 dirty slots, half load, 64 workers per bitset word, dead run records outnumbering the live entries), and the
    oracle's answers cover every branch of the pick."""
    plan = build_plan(jump)
    steps = plan["steps"]
    names = [st[1] for st in steps if st[0] == "T"]
    assert set(TRANSITIONS) <= set(names)
    for i, st in enumerate(steps):
        if st[0] == "T":
            assert steps[i - 1][0] == "submit" and steps[i + 1][0] == "submit", (i, st[1])
    # replay the model to read off what each transition did
    m = IndexModel()
    stats = {}
    for _ in range(W0):
        m.intern()
    for op, w, blocks in plan["init"]:
        m.store(w, blocks)
    for st in steps:
        if st[0] != "T":
            continue
        m.begin()
        for op, a, b in st[2]:
            if op == "stored":
                m.store(a, b)
            elif op == "removed":
                m.remove(a, b)
            elif op in ("cleared", "remove_worker"):
                m.clear(a)
            elif op == "intern":
                m.intern()
        stats.setdefault(st[1], dict(m.t, live_after=m.live(), tombs_after=m.tombs, cap_after=m.cap, words_after=m.words))
    sc, full, grow = stats["scatter"], stats["full"], stats["grow"]
    # scatter: few slots, no growth, a Multi entry at position 1, keys killed and stored again
    assert sc["touched"] < sc["cap_before"] // 8 and not sc["grew"] and sc["multi1"] and sc["killed"] and sc["reborn"]
    assert (sc["live_before"] + sc["tombs_before"] + sc["new_keys"]) * 2 < sc["cap_before"]
    # full: more than 1/8 of the slots dirty, no growth (live + every tombstone stay under half load)
    assert full["touched"] > full["cap_before"] // 8 and full["new_keys"] == 0 and full["killed"] > 64
    assert (full["live_after"] + full["tombs_after"]) * 2 < full["cap_before"] == 1024
    # grow: more than half of the 1024 slots live → a rebuild into a larger table for certain
    assert grow["cap_before"] == 1024 and grow["live_after"] * 2 > 1024 and grow["grew"]
    it = stats["intern65"]
    assert it["words_before"] == 1 and it["words_after"] == 2 and it["widened"]
    rows = stats["rows"]
    assert rows["words_after"] == 2 and rows["touched"] < rows["cap_before"] // 8 and rows["new_keys"] == 0 and not rows["grew"]
    cp = stats["compact"]   # runs_.size() - live > max(live, 1024) and runs_.size() ≥ 2 × the records kept at the last compaction
    assert cp["dead_records"] - 2 * MAX_BLOCKS > 2 * cp["records_before"] + 2 * m.max_live + 1024
    # slices: 64 → 70 workers, then 71 entries with a duplicate URL
    slices = [a for st in steps if st[0] == "T" for op, a, _ in st[2] if op == "slice"]
    assert [len(s) for s in slices] == [W_ALL, W_ALL + 1] and len(set(slices[1])) == W_ALL
    # requests: every kind, more than 32 blocks, empty, submissions that grow and shrink, offsets that do not start at 0
    subs = [st for st in steps if st[0] == "submit"]
    lens = [len(r) for st in subs for r in st[1]]
    assert 0 in lens and max(lens) > 32 * BS and any(0 < n < BS for n in lens)
    ns = [len(st[1]) for st in subs]
    assert 0 in ns and max(ns) >= 200 and any(a > b for a, b in zip(ns, ns[1:])) and any(st[2] > 0 for st in subs)
    want, _ = run_oracle(jump)
    br = set().union(*[set(e[1][1].tolist()) for e in want])
    assert {NO_HEALTHY, IMBALANCED, OVERLAP, MIN_LOAD} <= br
    assert sum(int((e[1][1] == OVERLAP).sum()) for e in want) > 200


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------

def _lib():
    from smg_b200 import _lib as L
    return L.load()


class Host:
    """Host output buffers of one submission, pageable (numpy) or pinned (smgx_alloc_pinned), poisoned."""

    def __init__(self, n, pinned, keep):
        self.n, self.pinned = n, pinned
        m = max(n, 1)
        if pinned:
            L = _lib()
            self.p_out, self.p_info = L.smgx_alloc_pinned(m * 4), L.smgx_alloc_pinned(m * INFO.itemsize)
            assert self.p_out and self.p_info
            keep.extend([self.p_out, self.p_info])
            self.out = np.frombuffer((C.c_int32 * m).from_address(self.p_out), np.int32)
            self.info = np.frombuffer((C.c_uint8 * (m * INFO.itemsize)).from_address(self.p_info), np.uint8).view(INFO)
            self.out[:] = POISON
            self.info.view(np.uint8)[:] = INFO_POISON
        else:
            self.out, self.info = np.full(m, POISON, np.int32), poisoned_info(n)

    def ptrs(self):
        return self.out.ctypes.data_as(C.c_void_p), self.info.ctypes.data_as(C.c_void_p)


def padded(reqs, pad, text=False):
    """Ragged requests with `pad` elements of poison before offsets[0]."""
    if text:
        blob = [t.encode() for t in reqs]
        data = np.frombuffer(b"\xa5" * pad + b"".join(blob) + b"\0", np.uint8).copy()
        lens = [len(b) for b in blob]
    else:
        tokens, _, lens = ragged(reqs)
        data = np.concatenate([np.full(pad, TOKEN_POISON, np.uint32), tokens, np.zeros(1, np.uint32)])
    offsets = np.zeros(len(reqs) + 1, np.uint32)
    offsets[0] = pad
    np.cumsum(lens, out=offsets[1:])
    offsets[1:] += pad
    return data, offsets


class Run:
    """One GPU policy driven through a plan."""

    def __init__(self, plan, jump, max_tokens=MAX_TOKENS, tokenizer=False):
        self.pol, self.ws, self.ix = gpu_policy(plan["urls"][:W0], jump, max_tokens)
        self.h, self.L = self.pol._h, _lib()
        self.slice = tuple(plan["urls"][:W0])
        self.depth = self.L.smgx_pipeline_depth(self.h.p)
        self.busy = [None] * self.depth    # lane → ticket (host-buffer submissions hold a lane until waited)
        self.pinned = []
        if tokenizer:
            import json
            g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bpe_vectors.json")))
            self.pol.load_tiktoken_tokenizer(VOCAB_FILE, g["specials"])
        apply_ops(self.ix, plan["init"])

    def close(self):
        self.h.call("smgx_synchronize")
        for p in self.pinned:
            self.L.smgx_free_pinned(p)
        self.pinned = []

    def set_slice(self, urls):
        from smg_b200 import BasicWorker
        self.slice = tuple(urls)
        self.ws = [BasicWorker(u) for u in urls]

    def push_fleet(self, fleet):
        self.model = set_fleet(self.pol, self.ws, fleet)

    def hold(self, lane):
        self.h.call("smgx_stream_hold", lane, HOLD_US)

    def free_lane(self):
        return self.busy.index(None)

    def submit(self, kind, reqs, pad, pinned):
        """submit_tokens / submit_text with poisoned outputs on the lane it will take, held first → (ticket, lane, Host, inputs)."""
        lane = self.free_lane()
        self.hold(lane)
        text = kind == "text"
        data, offsets = padded(reqs, pad, text)
        host = Host(len(reqs), pinned, self.pinned)
        out, info = host.ptrs()
        t = C.c_uint64()
        fn = "smgx_submit_text" if text else "smgx_submit_tokens"
        self.h.call(fn, self.model, data.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), len(reqs), out, info, C.byref(t))
        self.busy[lane] = t.value
        return dict(ticket=t.value, lane=lane, host=host, keep=(data, offsets))

    def wait(self, sub):
        self.h.call("smgx_wait", sub["ticket"])
        self.busy[sub["lane"]] = None


def drain(run, inflight, order, keep_last):
    """Wait for the submissions in flight in `order` (submission / reverse / interleaved), all but the newest if keep_last."""
    todo = inflight[:-1] if keep_last else inflight[:]
    if order == "reverse":
        todo = todo[::-1]
    elif order == "interleaved":
        todo = todo[1::2] + todo[0::2]
    done = []
    for s in todo:
        run.wait(s)
        done.append(s)
    for s in done:
        inflight.remove(s)
    return done


def run_host_plan(jump, kind, pinned, order):
    """The plan through smgx_submit_tokens / smgx_submit_text, up to depth tickets in flight → (results in submission order, processed)."""
    text_seed = 1 if kind == "text" else None
    plan = build_plan(jump, text_seed)
    texts = plan_texts(plan) if text_seed is not None else None
    run = Run(plan, jump, tokenizer=kind == "text")
    run.push_fleet(INITIAL_FLEET)
    try:
        subs, inflight = [], []
        for k, st in enumerate(plan["steps"]):
            if st[0] == "T":
                assert inflight, "a transition must find a submission in flight"
                apply_plan_ops(run, st[2], gpu=True)
                continue
            if len(inflight) == run.depth:
                drain(run, inflight, order, keep_last=True)
            reqs = texts[k][0] if texts else st[1]
            sub = run.submit(kind, reqs, st[2], pinned)
            sub["k"] = k
            subs.append(sub)
            inflight.append(sub)
            if len(inflight) == run.depth:   # keep the newest in flight over the next transition
                drain(run, inflight, order, keep_last=True)
        drain(run, inflight, order, keep_last=False)
        processed = run.pol.take_processed(n=len(run.slice))
        return [(s["k"], s["host"].out[:s["host"].n].copy(), s["host"].info[:s["host"].n].copy()) for s in subs], processed
    finally:
        run.close()


def run_device_plan(jump, many):
    """The plan through smgx_select_batch_tokens_device on lanes 0-3 in turn (or smgx_select_many_tokens_device, each submission
    split into up to three batches), never synchronising until the end → results in submission order."""
    plan = build_plan(jump)
    run = Run(plan, jump)
    run.push_fleet(INITIAL_FLEET)
    dev = Device(run.pol)
    reads, lane = [], 0
    try:
        for k, st in enumerate(plan["steps"]):
            if st[0] == "T":
                apply_plan_ops(run, st[2], gpu=True)
                continue
            reqs, pad = st[1], st[2]
            n = len(reqs)
            if not many:
                data, offsets = padded(reqs, pad)
                d_out, d_info = dev.put(np.full(max(n, 1), POISON, np.int32)), dev.put(poisoned_info(n))
                run.hold(lane)
                run.h.call("smgx_select_batch_tokens_device", run.model, lane, dev.put(data), dev.put(offsets), n, 0, d_out, d_info)
                reads.append((k, [(0, n, d_out, d_info)]))
                lane = (lane + 1) % run.depth
                continue
            cuts = sorted({0, n, n // 3, (2 * n) // 3})
            parts = [(a, b) for a, b in zip(cuts, cuts[1:])] + [(n, n)]   # the last batch is empty
            tok, off, outs = [], [], []
            for a, b in parts:
                data, offsets = padded(reqs[a:b], pad)
                tok.append(dev.put(data)); off.append(dev.put(offsets)); outs.append(dev.put(np.full(max(b - a, 1), POISON, np.int32)))
            for j in range(min(len(parts), run.depth)):
                run.hold(j)
            nb = len(parts)
            vp = C.c_void_p * nb
            run.h.call("smgx_select_many_tokens_device", run.model, nb, vp(*tok), vp(*off), (C.c_uint32 * nb)(*[b - a for a, b in parts]), 0,
                       vp(*outs))
            reads.append((k, [(a, b, p, None) for (a, b), p in zip(parts, outs)]))
        run.h.call("smgx_synchronize")
        res = []
        for k, parts in reads:
            n = sum(b - a for a, b, _, _ in parts)
            out, info = np.full(n, POISON, np.int32), None
            for a, b, p, pi in parts:
                got = dev.get(p, np.int32, max(b - a, 1))
                assert b > a or got[0] == POISON, "an empty batch had an output written"
                out[a:b] = got[:b - a]
                if pi is not None:
                    info = dev.get(pi, np.uint8, n * INFO.itemsize).view(INFO)
            res.append((k, out, info))
        return res
    finally:
        dev.free()
        run.close()


def check_tree(tag, idx, info, lens, want, tree_matched=None):
    """check() for submissions that may take the token-tree path: on the imbalanced branch `matched` is the tree match in tokens, the
    oracle's (or `tree_matched` where the tree update is applied later than the oracle applied it)."""
    oidx, obr, oma = want
    imb = np.asarray(obr) == IMBALANCED
    if info is not None and imb.any():
        exp = np.asarray(oma if tree_matched is None else tree_matched, np.int64)
        assert np.array_equal(info["matched"][imb].astype(np.int64), exp[imb]), f"{tag}: tree match of the imbalanced picks differs"
        info = info.copy()
        info["matched"][imb] = 0
    check(tag, idx, info, lens, want)


def check_results(tag, got, want, tree=False):
    by_k = {k: (w, lens) for k, w, lens in want}
    assert [k for k, _, _ in got] == [k for k, _, _ in want]
    for k, out, info in got:
        w, lens = by_k[k]
        (check_tree if tree else check)(f"{tag}, step {k} (n = {len(lens)})", out, info, lens, w)


@pytest.mark.gpu
@pytest.mark.parametrize("transport", ["submit_tokens", "submit_text", "device_lanes", "many"])
@pytest.mark.parametrize("jump", [64, 8])
def test_in_flight_batches_see_their_submission_state(jump, transport):
    """Every submission equals the oracle after exactly the transitions before it, bit for bit (picks, matched, input, branch), whatever
    is still in flight when the state changes and whatever order the tickets are waited in; pageable and pinned outputs."""
    if transport in ("device_lanes", "many"):
        want, _ = run_oracle(jump)
        check_results(f"{transport}, jump {jump}", run_device_plan(jump, transport == "many"), want)
        return
    kind = "text" if transport == "submit_text" else "tokens"
    want, processed = run_oracle(jump, 1 if kind == "text" else None)
    for pinned, order in [(False, "submission"), (True, "reverse"), (True, "interleaved")]:
        got, got_processed = run_host_plan(jump, kind, pinned, order)
        check_results(f"{transport}, jump {jump}, {'pinned' if pinned else 'pageable'}, {order}", got, want, tree=True)
        assert np.array_equal(got_processed, processed), (pinned, order)


# ---- lane bookkeeping, mapped submissions, mode switches, load feedback, processed counts, other policies -------------------------

def small_world(W=16, jump=64, seed=3, tokenizer=False):
    """A GPU policy and its oracle on the same index: W workers, 24 stored sequences → (pol, ws, ix, op, oix, seqs, rng)."""
    urls = synth.worker_urls(W)
    pol, ws, ix = gpu_policy(urls, jump, MAX_TOKENS)
    op, oix = oracle_policy(urls, jump)
    if tokenizer:
        import json
        g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bpe_vectors.json")))
        pol.load_tiktoken_tokenizer(VOCAB_FILE, g["specials"])
    rng = np.random.default_rng(seed)
    seqs = [np.asarray(s, np.uint32) for s in synth.gen_sequences(24, 40 * BS, 900 + seed)]
    ops = []
    for k, s in enumerate(seqs):
        hs = orc.compute_request_content_hashes(s, BS)
        ops.append(("stored", k % W, [(10_000 * (k + 1) + i, h) for i, h in enumerate(hs)]))
    apply_ops(ix, ops); apply_ops(oix, ops)
    return pol, ws, ix, op, oix, seqs, rng


def mixed_requests(rng, seqs, n):
    out = []
    for _ in range(n):
        s = seqs[int(rng.integers(0, len(seqs)))]
        r = rng.random()
        if r < 0.4:
            out.append(s[:int(rng.integers(1, 41)) * BS].copy())
        elif r < 0.7:
            out.append(np.concatenate([s[:int(rng.integers(1, 20)) * BS], rng.integers(0, synth.VOCAB, size=int(rng.integers(1, 200)), dtype=np.uint32)]))
        else:
            out.append(rng.integers(0, synth.VOCAB, size=int(rng.integers(0, 300)), dtype=np.uint32))
    return out


def oracle_pick(op, reqs, feedback=False):
    tokens, offsets, lens = ragged(reqs)
    if not reqs:
        return (np.zeros(0, np.int32), np.zeros(0, np.uint8), np.zeros(0, np.uint32)), lens
    fn = op.select_batch_tokens_feedback if feedback else op.select_batch_tokens
    r = fn(tokens, offsets.astype(np.uint64))
    return (np.asarray(r[0]), np.asarray(r[1]), np.asarray(r[2])), lens


def push(pol, ws, op, fleet):
    op.set_state(*fleet)
    return set_fleet(pol, ws, fleet)


def status_of(fn):
    from smg_b200 import SmgxError
    try:
        fn()
    except SmgxError as e:
        return e.code
    return 0


def tree_entries(pol):
    return pol.token_tree().entries()


def same_tree(a, b, timestamps=True):
    """Two token trees' entries hold the same paths and tenants, with the tenants' timestamps in the same order.  Timestamps are compared
    by rank: the oracle's clock is shared by every oracle policy of the process, the library's by the trees of one policy."""
    def ranked(entries):
        ts = {t: i for i, t in enumerate(sorted({t for _, ten in entries for _, t in ten}))}
        return sorted((tuple(toks), tuple(sorted((name, ts[t] if timestamps else 0) for name, t in ten))) for toks, ten in entries)
    return ranked(a) == ranked(b)


class Tickets:
    """Host-buffer submissions on one policy with the lane each takes held first."""

    def __init__(self, pol, model, pinned=True):
        self.pol, self.h, self.model, self.pinned, self.keep = pol, pol._h, model, pinned, []
        self.busy = [None] * _lib().smgx_pipeline_depth(self.h.p)

    def submit(self, reqs, pad=0, text=False, hold=True):
        lane = self.busy.index(None) if None in self.busy else None
        if hold and lane is not None:
            self.h.call("smgx_stream_hold", lane, HOLD_US)
        data, offsets = padded(reqs, pad, text)
        host = Host(len(reqs), self.pinned, self.keep)
        out, info = host.ptrs()
        t = C.c_uint64()
        self.h.call("smgx_submit_text" if text else "smgx_submit_tokens", self.model, data.ctypes.data_as(C.c_void_p),
                    offsets.ctypes.data_as(C.c_void_p), len(reqs), out, info, C.byref(t))
        self.busy[lane] = t.value
        return dict(ticket=t.value, lane=lane, host=host, inputs=(data, offsets), n=len(reqs))

    def wait(self, s):
        self.h.call("smgx_wait", s["ticket"])
        self.busy[s["lane"]] = None
        return s["host"].out[:s["n"]].copy(), s["host"].info[:s["n"]].copy()

    def close(self):
        self.h.call("smgx_synchronize")
        for p in self.keep:
            _lib().smgx_free_pinned(p)
        self.keep = []


@pytest.mark.gpu
def test_lane_bookkeeping():
    """SMGX_BUSY at depth + 1 changes nothing (no tree insert, nothing counted) and a retry after one wait succeeds; an unknown or
    twice-waited ticket is SMGX_INVALID_ARGUMENT; n = 0 gives a ticket that can be waited for; a lane reused after a wait returns the
    new batch, not a remnant of the old one."""
    pol, ws, ix, op, oix, seqs, rng = small_world()
    W = len(ws)
    balanced = (rng.integers(0, 10, size=W).astype(np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
    model = push(pol, ws, op, balanced)
    T = Tickets(pol, model)
    try:
        depth = len(T.busy)
        batches = [mixed_requests(rng, seqs, n) for n in (200, 30, 7, 90)]
        subs = [T.submit(b) for b in batches[:depth]]
        wants = [oracle_pick(op, b) for b in batches[:depth]]
        # the (depth + 1)-th submission, on an imbalanced fleet: it would take the token tree path and insert
        imb = (balanced[0].copy(), balanced[1], balanced[2])
        imb[0][3] = 500
        T.model = push(pol, ws, op, imb)
        before = tree_entries(pol)
        extra = mixed_requests(rng, seqs, 12)
        assert status_of(lambda: T.submit(extra, hold=False)) == SMGX_BUSY
        assert tree_entries(pol) == before
        got = T.wait(subs[1])
        check("ticket 1", *got, wants[1][1], wants[1][0])
        retry = T.submit(extra)   # tree path: completes inside the call, on the lane just freed
        want_extra = oracle_pick(op, extra)
        assert tree_entries(pol) != before
        for i in (0, 2, 3):
            check(f"ticket {i}", *T.wait(subs[i]), wants[i][1], wants[i][0])
        check_tree("retry", *T.wait(retry), want_extra[1], want_extra[0])
        assert set(want_extra[0][1].tolist()) == {IMBALANCED}
        # unknown and twice-waited tickets
        assert status_of(lambda: pol._h.call("smgx_wait", retry["ticket"])) == SMGX_INVALID_ARGUMENT
        assert status_of(lambda: pol._h.call("smgx_wait", 1 << 60)) == SMGX_INVALID_ARGUMENT
        # counted: the four tickets and the retry, never the refused submissions
        T.model = push(pol, ws, op, balanced)
        assert np.array_equal(pol.take_processed(n=W), np.array([op.processed(i) for i in range(W)], np.uint64))
        # n = 0: a ticket that can be waited for, once
        z = T.submit([], pad=3)
        T.wait(z)
        assert status_of(lambda: pol._h.call("smgx_wait", z["ticket"])) == SMGX_INVALID_ARGUMENT
        # lane reuse: a large batch, waited; a small batch on the same lane returns its own picks and leaves the rest of its buffer alone
        big = mixed_requests(rng, seqs, 300)
        s = T.submit(big)
        lane_big = s["lane"]
        check("big", *T.wait(s), oracle_pick(op, big)[1], oracle_pick(op, big)[0])
        small = mixed_requests(rng, seqs, 5)
        s = T.submit(small, pad=2)
        assert s["lane"] == lane_big
        check("small after big", *T.wait(s), oracle_pick(op, small)[1], oracle_pick(op, small)[0])
        assert s["host"].out[5:].size == 0 or (s["host"].out[5:] == POISON).all()
    finally:
        T.close()


def check_pick(tag, got, want_lens):
    (out, info), (want, lens) = got, want_lens
    check(tag, out, info, lens, want)


@pytest.mark.gpu
def test_mapped_submissions_between_host_tickets():
    """Four host-buffer tickets hold every lane; then 4k mapped submissions go out round-robin over those busy lanes, with index and fleet
    changes in between.  Each mapped batch and each ticket equals the oracle at its own submission.  In tree mode (imbalanced fleet) a
    mapped submission is SMGX_NOT_FOUND and changes neither the tree nor the tickets."""
    pol, ws, ix, op, oix, seqs, rng = small_world(seed=5)
    W = len(ws)
    L = _lib()
    fleet = (rng.integers(0, 10, size=W).astype(np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
    model = push(pol, ws, op, fleet)
    T = Tickets(pol, model)
    pinned = []
    try:
        host_reqs = [mixed_requests(rng, seqs, n) for n in (40, 9, 120, 3)]
        subs = [T.submit(r) for r in host_reqs]
        wants = [oracle_pick(op, r) for r in host_reqs]
        depth = len(subs)
        mapped = []
        sid = 900_000
        for j in range(4 * depth):
            if j % 3 == 1:   # scatter: a new sequence and an eviction
                s = seqs[int(rng.integers(0, len(seqs)))]
                hs = orc.compute_request_content_hashes(s[:10 * BS], BS)
                w = int(rng.integers(0, W))
                ops = [("stored", w, [(sid + i, h) for i, h in enumerate(hs)]), ("removed", w, [sid + 7, sid + 8, sid + 9])]
                sid += 100
                apply_ops(ix, ops); apply_ops(oix, ops)
            elif j % 3 == 2:
                fleet = (rng.integers(0, 10, size=W).astype(np.uint64), (rng.random(W) > 0.1).astype(np.uint8), np.ones(W, np.uint8))
                model = push(pol, ws, op, fleet)
            reqs = mixed_requests(rng, seqs, int(rng.integers(1, 24)))
            data, offsets = padded(reqs, int(rng.integers(0, 4)))
            n = len(reqs)
            bufs = [L.smgx_alloc_pinned(max(data.nbytes, 4)), L.smgx_alloc_pinned(offsets.nbytes), L.smgx_alloc_pinned(n * 4),
                    L.smgx_alloc_pinned(n * INFO.itemsize), L.smgx_alloc_pinned(8)]
            assert all(bufs)
            pinned.extend(bufs)
            C.memmove(bufs[0], data.ctypes.data, data.nbytes)
            C.memmove(bufs[1], offsets.ctypes.data, offsets.nbytes)
            out = np.frombuffer((C.c_int32 * n).from_address(bufs[2]), np.int32)
            info = np.frombuffer((C.c_uint8 * (n * INFO.itemsize)).from_address(bufs[3]), np.uint8).view(INFO)
            flag = np.frombuffer((C.c_uint64 * 1).from_address(bufs[4]), np.uint64)
            out[:] = POISON
            info.view(np.uint8)[:] = INFO_POISON
            flag[0] = 0
            pol._h.call("smgx_submit_tokens_mapped", model, bufs[0], bufs[1], n, 0, bufs[2], bufs[3], bufs[4], j + 1)
            mapped.append((j, out, info, flag, oracle_pick(op, reqs)))
        deadline = time.monotonic() + 60
        for j, out, info, flag, (want, lens) in mapped:
            while int(flag[0]) != j + 1:
                assert time.monotonic() < deadline, f"mapped submission {j}: done flag never raised"
                time.sleep(0.0005)
            check(f"mapped {j}", out.copy(), info.copy(), lens, want)
        for i, s in enumerate(subs):
            check(f"ticket {i}", *T.wait(s), wants[i][1], wants[i][0])
        # tree mode: refused, nothing changes
        subs = [T.submit(r) for r in host_reqs[:2]]
        wants = [oracle_pick(op, r) for r in host_reqs[:2]]
        imb = (fleet[0].copy(), np.ones(W, np.uint8), np.ones(W, np.uint8))
        imb[0][2] = 900
        model = push(pol, ws, op, imb)
        before = tree_entries(pol)
        data, offsets = padded(host_reqs[1], 0)
        bufs = [L.smgx_alloc_pinned(data.nbytes), L.smgx_alloc_pinned(offsets.nbytes), L.smgx_alloc_pinned(64), L.smgx_alloc_pinned(64 * INFO.itemsize),
                L.smgx_alloc_pinned(8)]
        pinned.extend(bufs)
        C.memmove(bufs[0], data.ctypes.data, data.nbytes)
        C.memmove(bufs[1], offsets.ctypes.data, offsets.nbytes)
        assert status_of(lambda: pol._h.call("smgx_submit_tokens_mapped", model, bufs[0], bufs[1], len(host_reqs[1]), 0, bufs[2], bufs[3], bufs[4], 1)) == SMGX_NOT_FOUND
        assert tree_entries(pol) == before
        for i, s in enumerate(subs):
            check(f"ticket {i} after the refusal", *T.wait(s), wants[i][1], wants[i][0])
    finally:
        pol._h.call("smgx_synchronize")
        T.close()
        for p in pinned:
            L.smgx_free_pinned(p)


@pytest.mark.gpu
def test_mode_switch_with_a_ticket_in_flight():
    """An event-mode ticket with pinned outputs is in flight on lane 0 while the indexer is cleared (the token tree takes over:
    smgx_submit_tokens and smgx_submit_text, whose tree walk runs on lane 0) and, once blocks are stored again, an imbalanced fleet with a
    non-empty tree sends smgx_submit_tokens down the tree path.  The ticket's picks and info are intact, the tree-mode picks equal the
    oracle and the token tree equals the oracle's."""
    enc = text_encoding()
    pol, ws, ix, op, oix, seqs, rng = small_world(seed=11, tokenizer=True)
    W = len(ws)
    fleet = (rng.integers(0, 10, size=W).astype(np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
    model = push(pol, ws, op, fleet)
    T = Tickets(pol, model)
    try:
        reqs0 = mixed_requests(rng, seqs, 150)
        t0 = T.submit(reqs0, pad=3)
        assert t0["lane"] == 0
        want0 = oracle_pick(op, reqs0)
        for w in range(W):
            ix.apply_cleared(w); oix.apply_cleared(w)
        assert ix.current_size() == 0 and oix.current_size() == 0
        texts = [ascii_text(rng, int(rng.integers(0, 400))) for _ in range(20)] + ["", "the route"]
        tree_reqs = mixed_requests(rng, seqs, 30)
        got = []
        s1 = T.submit(tree_reqs, pad=1)                 # tree mode, on lane 1
        got.append(("tokens", T.wait(s1), oracle_pick(op, tree_reqs)))
        s2 = T.submit(texts, pad=2, text=True)          # tree mode; the tree walk runs on lane 0 with the ticket still in flight
        ref = [np.asarray(enc.encode(t, allowed_special="all"), np.uint32) for t in texts]
        got.append(("text", T.wait(s2), oracle_pick(op, ref)))
        # blocks again (event mode), then an imbalanced fleet with a non-empty token tree: the tree path of submit_host
        ops = [("stored", 3, [(777_000 + i, h) for i, h in enumerate(orc.compute_request_content_hashes(seqs[5], BS))])]
        apply_ops(ix, ops); apply_ops(oix, ops)
        imb = (fleet[0].copy(), fleet[1], fleet[2])
        imb[0][6] = 700
        T.model = push(pol, ws, op, imb)
        imb_reqs = tree_reqs[:10] + mixed_requests(rng, seqs, 10)
        s3 = T.submit(imb_reqs)
        got.append(("imbalanced", T.wait(s3), oracle_pick(op, imb_reqs)))
        check("in-flight event ticket", *T.wait(t0), want0[1], want0[0])
        for tag, (out, info), (want, lens) in got:
            assert not (out == POISON).any(), tag
            assert np.array_equal(out, want[0]), (tag, np.nonzero(out != want[0])[0][:5])
            assert np.array_equal(info["branch"], want[1]), tag
            assert np.array_equal(info["input"], lens), tag
            assert np.array_equal(info["matched"], want[2]), tag
        assert {TREE_MATCH, TREE_MIN_LOAD} & set(got[0][2][0][1].tolist())
        assert set(got[2][2][0][1].tolist()) == {IMBALANCED}
        assert same_tree(tree_entries(pol), op.token_tree().entries())
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["submission", "reverse"])
def test_load_feedback_through_submissions(order):
    """SMGX_FEEDBACK_CACHE_AWARE with several tickets in flight, the fleet changed before each: every ticket equals
    select_batch_tokens_feedback on its own submission's snapshot.  The token-tree update owed by the picks that took the imbalanced
    branch is applied when the ticket is waited for, so the tree equals an oracle tree that received those requests in wait order."""
    pol, ws, ix, op, oix, seqs, rng = small_world(seed=17)
    W = len(ws)
    pol._h.call("smgx_set_load_feedback_policies", 1)
    tree_op = orc.CacheAwarePolicy(eviction_interval_secs=0, cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=BS)
    tree_op.set_workers(synth.worker_urls(W))
    fleet = (np.full(W, 5, np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
    T = Tickets(pol, push(pol, ws, op, fleet))
    try:
        subs = []
        for k in range(4):
            loads = rng.integers(0, 20, size=W).astype(np.uint64)
            if k % 2 == 0:
                loads[int(rng.integers(0, W))] = 300 + 40 * k   # imbalanced: the first picks take the imbalanced branch
            healthy = (rng.random(W) > 0.1).astype(np.uint8)
            T.model = push(pol, ws, op, (loads, healthy, np.ones(W, np.uint8)))
            reqs = mixed_requests(rng, seqs, int(rng.integers(40, 160)))
            subs.append((T.submit(reqs, pad=k), reqs, oracle_pick(op, reqs, feedback=True)))
        waits = subs if order == "submission" else subs[::-1]
        n_imb = 0
        for k, (s, reqs, (want, lens)) in enumerate(waits):
            out, info = T.wait(s)
            tree_matched = np.zeros(len(reqs), np.int64)
            for i in np.nonzero((want[1] == IMBALANCED) & (want[0] >= 0))[0]:   # the deferred tree update, in wait order
                forced = np.full(W, 1000, np.uint64)
                forced[int(want[0][i])] = 0
                tree_op.set_state(forced, np.ones(W, np.uint8), np.ones(W, np.uint8))
                d = tree_op.select_worker(tokens=reqs[i])
                assert d.idx == int(want[0][i]) and d.branch == "imbalanced_min_load"
                tree_matched[i] = d.matched
                n_imb += 1
            check_tree(f"ticket {k} ({order})", out, info, lens, want, tree_matched)
        assert n_imb > 10
        assert same_tree(tree_entries(pol), tree_op.token_tree().entries(), timestamps=False)
    finally:
        T.close()


@pytest.mark.gpu
def test_processed_counts_of_pipelined_calls():
    """smgx_take_processed after every wait equals the oracle's processed(i) for every slice index, across submit_tokens, submit_text
    and the tree path (mapped submissions leave counting to the caller).  A ticket is credited when it is waited for: a take between
    submit and wait does not see it, the next take does.  A ticket submitted before smgx_set_workers replaced the slice is not credited
    to the new slice (known answer: every count is 0 after the replacement)."""
    enc = text_encoding()
    pol, ws, ix, op, oix, seqs, rng = small_world(seed=23, tokenizer=True)
    W = len(ws)
    fleet = (rng.integers(0, 10, size=W).astype(np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
    T = Tickets(pol, push(pol, ws, op, fleet))
    try:
        a = mixed_requests(rng, seqs, 60)
        sa = T.submit(a)
        want_a = oracle_pick(op, a)
        assert np.array_equal(pol.take_processed(n=W), np.zeros(W, np.uint64))   # not waited yet: nothing counted
        T.wait(sa)
        base = np.array([op.processed(i) for i in range(W)], np.uint64)
        assert base.sum() == (want_a[0][0] >= 0).sum() > 0 and np.array_equal(pol.take_processed(n=W), base)
        # tokens, text and the tree path, waited in mixed order
        texts = [ascii_text(rng, int(rng.integers(0, 300))) for _ in range(25)]
        b, c = mixed_requests(rng, seqs, 80), mixed_requests(rng, seqs, 30)
        sb = T.submit(b)
        sc_ = T.submit(texts, text=True)
        oracle_pick(op, b)
        oracle_pick(op, [np.asarray(enc.encode(t, allowed_special="all"), np.uint32) for t in texts])
        imb = (fleet[0].copy(), fleet[1], fleet[2])
        imb[0][1] = 600
        T.model = push(pol, ws, op, imb)
        sd = T.submit(c)   # tree path: counted inside the call
        oracle_pick(op, c)
        T.wait(sc_); T.wait(sd); T.wait(sb)
        now = np.array([op.processed(i) for i in range(W)], np.uint64)
        assert np.array_equal(pol.take_processed(n=W), now - base)
        # a ticket in flight while smgx_set_workers replaces the slice
        T.model = push(pol, ws, op, fleet)
        se = T.submit(mixed_requests(rng, seqs, 50))
        from smg_b200 import BasicWorker
        urls2 = synth.worker_urls(W)[::-1]
        ws2 = [BasicWorker(u) for u in urls2]
        op.set_workers(urls2)
        T.model = push(pol, ws2, op, fleet)
        T.wait(se)
        assert np.array_equal(pol.take_processed(n=W), np.zeros(W, np.uint64))
        assert all(op.processed(i) == 0 for i in range(W))
    finally:
        T.close()


@pytest.mark.gpu
def test_other_policies_between_submissions():
    """With event tickets in flight on every lane: a device-resident prefix_hash call on lanes 0/1 left unsynchronised, then new loads and
    a new ring; a host-buffer prefix_hash call; a power_of_two and a consistent_hashing call.  Each equals its oracle and the event tickets
    are unchanged."""
    pol, ws, ix, op, oix, seqs, rng = small_world(seed=29)
    W = len(ws)
    urls = synth.worker_urls(W)
    loads = rng.integers(0, 30, size=W).astype(np.uint64)
    healthy = (rng.random(W) > 0.15).astype(np.uint8)
    fleet = (loads, healthy, np.ones(W, np.uint8))
    model = push(pol, ws, op, fleet)
    T = Tickets(pol, model)
    dev = Device(pol)
    try:
        ring_urls = urls[:12]
        pol._h.call("smgx_hash_ring_set", model, (C.c_char_p * len(ring_urls))(*[u.encode() for u in ring_urls]), len(ring_urls))
        ev = [mixed_requests(rng, seqs, n) for n in (70, 20, 150, 5)]
        subs = [T.submit(r) for r in ev]
        wants = [oracle_pick(op, r) for r in ev]
        ph = orc.PrefixHashPolicy()
        # device-resident prefix_hash, unsynchronised
        hot = seqs[0][:300]
        pf_reqs = [np.concatenate([hot if rng.random() < 0.5 else np.zeros(0, np.uint32), rng.integers(0, synth.VOCAB, size=int(rng.integers(1, 300)), dtype=np.uint32)]) for _ in range(120)]
        tokens, offsets, _ = ragged(pf_reqs)
        d_out = dev.put(np.full(len(pf_reqs), POISON, np.int32))
        vp = C.c_void_p * 1
        pol._h.call("smgx_prefix_hash_select_many_tokens_device", model, 1, vp(dev.put(tokens)), vp(dev.put(offsets)), (C.c_uint32 * 1)(len(pf_reqs)), vp(d_out))
        want_pf, _, _ = ph.select_batch(urls, loads, healthy, orc.HashRing(ring_urls), tokens, offsets.astype(np.uint64))
        # new loads and a new ring while it may still run
        loads2 = rng.integers(0, 30, size=W).astype(np.uint64)
        healthy2 = (rng.random(W) > 0.15).astype(np.uint8)
        fleet2 = (loads2, healthy2, np.ones(W, np.uint8))
        model = push(pol, ws, op, fleet2)
        ring2 = urls[4:]
        pol._h.call("smgx_hash_ring_set", model, (C.c_char_p * len(ring2))(*[u.encode() for u in ring2]), len(ring2))
        # host-buffer prefix_hash (staging on lane 0)
        h_reqs = pf_reqs[::-1][:80]
        tokens2, offsets2, _ = ragged(h_reqs)
        out2 = np.full(len(h_reqs), POISON, np.int32)
        info2 = poisoned_info(len(h_reqs))
        pol._h.call("smgx_prefix_hash_select_batch_tokens", model, tokens2.ctypes.data_as(C.c_void_p), offsets2.ctypes.data_as(C.c_void_p), len(h_reqs), None,
                    out2.ctypes.data_as(C.c_void_p), info2.ctypes.data_as(C.c_void_p))
        want2, wbr2, _ = ph.select_batch(urls, loads2, healthy2, orc.HashRing(ring2), tokens2, offsets2.astype(np.uint64))
        assert np.array_equal(out2, want2) and np.array_equal(info2["branch"], wbr2)
        # power_of_two
        n = 500
        seed = int(rng.integers(0, 2**63))
        p_out, p_pairs, p_metric = np.full(n, POISON, np.int32), np.full(2 * n, POISON, np.int32), np.zeros(n, np.uint8)
        pol._h.call("smgx_power_of_two_select_batch", model, n, seed, p_out.ctypes.data_as(C.c_void_p), p_pairs.ctypes.data_as(C.c_void_p),
                    p_metric.ctypes.data_as(C.c_void_p))
        oidx, opairs, ometric, _ = orc.PowerOfTwoPolicy().select_batch(urls, loads2, healthy2, np.ones(W, np.uint8), n, seed)
        assert np.array_equal(p_out, oidx) and np.array_equal(p_pairs.reshape(n, 2), opairs) and np.array_equal(p_metric, ometric)
        # consistent_hashing: routing keys, target workers and the random fallback
        hs = []
        for i in range(300):
            r = rng.random()
            if r < 0.4:
                hs.append([None, b"session-%d" % int(rng.integers(0, 50)), None, None, None])
            elif r < 0.6:
                hs.append([b"%d" % int(rng.integers(0, W + 2)), None, None, None, None])
            else:
                hs.append(None)
        blob, c_offs, present = ch.pack(hs)
        values = np.frombuffer(blob + b"\0", np.uint8).copy()
        c_offs, present = np.asarray(c_offs, np.uint32), np.asarray(present, np.uint8)
        seed2 = int(rng.integers(0, 2**63))
        c_out, c_br = np.full(300, POISON, np.int32), np.zeros(300, np.uint8)
        pol._h.call("smgx_consistent_hashing_select_batch", model, 300, values.ctypes.data_as(C.c_void_p), c_offs.ctypes.data_as(C.c_void_p),
                    present.ctypes.data_as(C.c_void_p), seed2, c_out.ctypes.data_as(C.c_void_p), c_br.ctypes.data_as(C.c_void_p), None)
        want_ch, _, _ = ch.select_batch(urls, healthy2.tolist(), ch.Ring(ring2), hs, seed2)
        assert c_out.tolist() == want_ch
        # the event tickets, then the device-resident prefix_hash result
        for i, s in enumerate(subs):
            check(f"ticket {i}", *T.wait(s), wants[i][1], wants[i][0])
        pol._h.call("smgx_synchronize")
        assert np.array_equal(dev.get(d_out, np.int32, len(pf_reqs)), want_pf)
    finally:
        dev.free()
        T.close()
