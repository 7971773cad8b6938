"""Launch sequences of the event-driven pick against the oracle.

The rest of the suite checks each implementation of the event-driven pick one call at a time.  Here every implementation serves a long
sequence of calls on one policy, mostly on stream lane 0, with totals that grow and shrink, index and fleet changes between calls, and
requests that take the generic search (more than 32 blocks, more than one jump, Multi entries).  The default pair hands those requests
from event_simple_kernel to event_slow_kernel through a per-lane device queue: its count and CTA exit counter must be zero again when a
launch ends, whatever the size of the next launch, or a later launch re-runs stale entries.

A Multi entry at position 0 cannot be built: the prefix hash of position 0 is its content hash, so every store of a block at position 0
carries the same prefix (event_tree.rs:338-342).  The sequences use position 1, the first position a drain reads, instead.

build_plan() makes a sequence from a seed alone and run_oracle() plays it on the oracle; the CPU test checks that a sequence contains what
the GPU tests rely on, so that an edit of the builder cannot quietly stop them reaching the queue."""
import ctypes as C
import functools
from contextlib import contextmanager

import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth

BS = 16
MAX_BLOCKS = 64                 # max_tokens_per_request = MAX_BLOCKS × BS
CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=BS)
POISON = -7
INFO_POISON = 0xA5
INFO = np.dtype([("matched", "<u4"), ("input", "<u4"), ("branch", "u1"), ("nodes", "u1"), ("reserved", "u1", 2)])
NO_HEALTHY, IMBALANCED, OVERLAP, MIN_LOAD = 0, 1, 2, 3

# every implementation that serves a plain pick: (event path, simple kernel, tile) for smgx_set_event_path / _event_simple / _fused_tile
IMPLS = {
    "simple": (1, 5, 0),    # the default: event_simple_kernel + event_slow_kernel
    "fused": (1, 0, 0),     # warp-per-request fused kernel
    "tile": (1, 0, 16),     # tiled kernel, from a total of 0 on
    "split": (0, 0, 0),     # hash kernel + search kernel
    "hs": (2, 0, 0),        # one launch: hash stream whose last CTA per group searches
    "stream": (3, 0, 0),    # persistent streaming kernel
}


@contextmanager
def selected(impl):
    """Select one implementation for the duration of the block; the defaults are restored whatever happens."""
    from smg_b200 import _lib
    L = _lib.load()
    path, simple, tile = IMPLS[impl]
    try:
        L.smgx_set_event_path(path, 4)
        L.smgx_set_event_simple(simple)
        L.smgx_set_fused_tile(tile, 0)
        yield
    finally:
        L.smgx_set_event_path(1, 4)
        L.smgx_set_event_simple(5)
        L.smgx_set_fused_tile(16, -1)


# ---- the sequence: requests, index and fleet changes, lanes (pure data, no GPU) ---------------------------------------------------

def queues(kind, nblk, jump):
    """Would event_simple_kernel hand this request to event_slow_kernel (on a healthy, balanced fleet)?"""
    return nblk > 32 or nblk - 1 > jump or kind.startswith("multi")


# (kind of call, lane, requests per batch, request mix, fleet).  Lane 0 starts small so that the growth to 200 and to 1000 reallocates
# its queue; "queued" calls queue every request and are followed by smaller totals, imbalanced and no-healthy calls.
SCHEDULE = [
    ("one", 0, [8], "mixed", "balanced"), ("one", 0, [3], "short", "balanced"), ("one", 0, [1], "queued", "balanced"),
    ("one", 0, [64], "queued", "balanced"), ("one", 0, [8], "short", "imbalanced"), ("one", 0, [8], "mixed", "balanced"),
    ("one", 0, [200], "mixed", "balanced"), ("one", 0, [16], "short", "none"), ("one", 1, [40], "mixed", "balanced"),
    ("one", 0, [120], "queued", "balanced"), ("one", 0, [5], "mixed", "one_down"), ("many", 0, [30, 0, 7, 50], "mixed", "balanced"),
    ("one", 0, [33], "mixed", "imbalanced"), ("one", 0, [300], "fits", "balanced"), ("one", 0, [12], "mixed", "balanced"),
    ("many", 0, [64, 64, 64], "fits", "balanced"), ("one", 0, [1000], "mixed", "balanced"), ("one", 0, [2], "queued", "balanced"),
    ("one", 0, [7], "short", "imbalanced"), ("one", 2, [25], "queued", "balanced"), ("one", 0, [90], "fits", "one_down"),
    ("many", 0, [5, 100, 1], "mixed", "balanced"), ("one", 0, [450], "queued", "balanced"), ("one", 0, [9], "mixed", "imbalanced"),
    ("one", 0, [9], "mixed", "balanced"), ("one", 0, [128], "fits", "balanced"), ("one", 3, [17], "mixed", "one_down"),
    ("one", 0, [640], "mixed", "balanced"), ("many", 0, [200, 0, 200], "fits", "balanced"), ("one", 0, [60], "queued", "one_down"),
    ("one", 0, [6], "mixed", "imbalanced"), ("one", 0, [256], "fits", "balanced"), ("one", 0, [31], "mixed", "balanced"),
    ("many", 0, [1, 2, 3, 4, 5, 6], "mixed", "balanced"), ("one", 0, [800], "queued", "balanced"), ("one", 0, [20], "short", "balanced"),
    ("one", 0, [500], "fits", "imbalanced"), ("one", 0, [70], "mixed", "one_down"), ("one", 1, [300], "mixed", "balanced"),
    ("one", 0, [3], "queued", "balanced"), ("one", 0, [100], "fits", "balanced"), ("one", 0, [48], "mixed", "imbalanced"),
    ("one", 0, [11], "mixed", "balanced"), ("many", 0, [32, 32], "fits", "balanced"),
]


@functools.lru_cache(maxsize=None)
def build_plan(jump, n_workers=16, seed=None):
    """A launch sequence for an indexer with this jump size.  → dict(urls, jump, init (index ops), steps); a step is dict(many, lane,
    cap (max_request_tokens, 0 = the policy's), batches (lists of token arrays), kinds (per request), ops (index changes applied before
    the call), fleet (loads, healthy, circuit_ok), mix (the request mix's name))."""
    rng = np.random.default_rng(jump if seed is None else seed)
    W = n_workers
    seqs = synth.gen_sequences(160, MAX_BLOCKS * BS, 100 + jump)   # 96 stored up front, the rest by later steps
    depth_of = {}
    sid = [1]
    removable = []   # (worker, blocks) stored by the population, candidates for apply_removed

    def store(w, tokens, depth, keep=True):
        hs = orc.compute_request_content_hashes(tokens[:depth * BS], BS)
        blocks = [(sid[0] + i, hs[i]) for i in range(depth)]
        sid[0] += depth
        if keep:
            removable.append((w, blocks))
        return ("stored", w, blocks)

    def noise(n):
        return rng.integers(0, synth.VOCAB, size=n, dtype=np.uint32)

    # Multi entries: the same block at the same position under two prefixes (as test_gpu_event_simple_shapes.py builds them)
    md, xd, mb, xb, mc, xc = synth.gen_sequences(6, 8 * BS, 200 + jump)
    xd[BS:2 * BS] = md[BS:2 * BS]              # (1, block 1 of md): md[:8] drains from 1 and meets it first
    xb[4 * BS:5 * BS] = mb[4 * BS:5 * BS]      # (4, block 4 of mb): inside the drain of mb[:8]
    xc[5 * BS:6 * BS] = mc[5 * BS:6 * BS]      # (5, block 5 of mc): the last position of mc[:6]
    init = [store(0, md, 8, False), store(1, md, 1, False), store(2, xd, 2, False),
            store(0, mb, 8, False), store(1, mb, 6, False), store(2, xb, 5, False),
            store(0, mc, 6, False), store(3, xc, 6, False)]
    multi = {"multi_first": md[:8 * BS], "multi_drain": mb[:8 * BS], "multi_last": mc[:6 * BS]}

    def store_population(s):
        for w in rng.choice(W, size=int(rng.integers(1, 4)), replace=False):
            d = int(rng.integers(1, MAX_BLOCKS + 1))
            depth_of[s] = max(depth_of.get(s, 0), d)
            yield store(int(w), seqs[s], d)
    for s in range(96):
        init.extend(store_population(s))
    next_seq = 96

    def request(kind, lim):
        """One request of this kind with at most `lim` full blocks."""
        s = int(rng.integers(0, next_seq))
        if kind == "tiny":
            r = seqs[s, :int(rng.integers(1, BS))].copy() if rng.random() < 0.5 else noise(int(rng.integers(1, BS)))
        elif kind in multi:
            r = multi[kind].copy()
        else:
            nblk = {"b1": 1, "b32": 32, "b33": 33, "long": int(rng.integers(40, MAX_BLOCKS + 1)),
                    "jumps": int(rng.integers(jump + 2, 33)) if jump + 2 <= 32 else 33}.get(kind)
            if kind == "hit":     # the whole stored depth of a sequence: a full hit
                nblk = depth_of[s]
            elif nblk is None:    # partial or novel
                nblk = int(rng.integers(1, MAX_BLOCKS + 1))
            nblk = min(nblk, lim)
            r = seqs[s, :nblk * BS].copy()
            if kind == "partial" and nblk > 1:
                k = int(rng.integers(1, nblk))
                r[k * BS:] = noise((nblk - k) * BS)
            elif kind == "novel":
                r = noise(nblk * BS)
        if rng.random() < 0.3 and kind != "tiny":   # a partial last block is not hashed
            r = np.concatenate([r, noise(int(rng.integers(1, BS)))])
        return r

    small = min(32, jump + 1)   # the tiled kernel needs max_blocks ≤ 32 and jump + 1 ≥ max_blocks; the streaming kernel ≤ 32
    every = ["tiny", "b1", "b32", "b33", "long", "hit", "partial", "novel", "multi_first", "multi_drain", "multi_last"]
    mixes = {
        "mixed": (every, MAX_BLOCKS),
        "queued": (["long", "b33", "multi_first", "multi_drain", "multi_last"] + (["jumps"] if jump + 2 <= 32 else []), MAX_BLOCKS),
        "short": (["tiny", "b1", "hit", "partial", "novel"], small),
        "fits": ([k for k in every if k not in ("b33", "long") and (k != "b32" or small >= 32)], small),
    }
    steps = []
    for i, (how, lane, ns, mix, fl) in enumerate(SCHEDULE):
        ops = []
        if i % 3 == 0 and i and next_seq < len(seqs):
            for s in range(next_seq, min(next_seq + 3, len(seqs))):
                ops.extend(store_population(s))
            next_seq = min(next_seq + 3, len(seqs))
        elif i % 3 == 1 and i > 1:
            for j in rng.choice(len(removable), size=2, replace=False):
                w, blocks = removable[j]
                if blocks:
                    cut = int(rng.integers(0, len(blocks)))   # evict the tail from `cut` on (cut = 0: the whole sequence)
                    ops.append(("removed", w, [b[0] for b in blocks[cut:]]))
                    removable[j] = (w, blocks[:cut])
        kinds_of, lim = mixes[mix]
        kinds = [[str(rng.choice(kinds_of)) for _ in range(n)] for n in ns]
        if mix == "queued":   # every shape that queues, whatever the batch size
            for ks in kinds:
                ks[:len(kinds_of)] = kinds_of[:len(ks)]
        batches = [[request(k, lim) for k in ks] for ks in kinds]
        loads = rng.integers(0, 21, size=W).astype(np.uint64)
        healthy, circuit = np.ones(W, np.uint8), np.ones(W, np.uint8)
        if fl == "imbalanced":
            loads[int(rng.integers(0, W))] = 300
        elif fl == "one_down":
            down, tripped = rng.choice(W, size=2, replace=False)
            healthy[down] = 0
            circuit[tripped] = 0
        elif fl == "none":
            healthy[:] = 0
        steps.append(dict(many=how == "many", lane=lane, cap=0 if lim == MAX_BLOCKS else lim * BS, batches=batches, kinds=kinds, ops=ops,
                          fleet=(loads, healthy, circuit), mix=mix))
    return dict(urls=synth.worker_urls(W), jump=jump, init=init, steps=steps)


def apply_ops(ix, ops):
    """Index changes, on the GPU policy's indexer or the oracle's."""
    for op, w, arg in ops:
        if op == "stored":
            ix.apply_stored(w, arg)
        else:
            ix.apply_removed(w, arg)


def ragged(reqs):
    lens = np.array([len(r) for r in reqs], np.uint32)
    offsets = np.zeros(len(reqs) + 1, np.uint32)
    np.cumsum(lens, out=offsets[1:])
    tokens = np.concatenate(reqs).astype(np.uint32) if len(reqs) else np.zeros(0, np.uint32)
    return tokens, offsets, lens


def oracle_policy(urls, jump):
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **CFG)
    op.set_workers(urls)
    oix = orc.PositionalIndexer(jump)
    op.attach_indexer("unknown", oix)
    op.set_block_size("unknown", BS)
    op.set_kv_event_monitor(True)
    for u in urls:
        oix.intern_worker(u)
    return op, oix


@functools.lru_cache(maxsize=None)
def run_oracle(jump):
    """The plan's expected answers: per step, per batch, (picks, branches, matched tokens)."""
    plan = build_plan(jump)
    op, oix = oracle_policy(plan["urls"], jump)
    apply_ops(oix, plan["init"])
    out = []
    for st in plan["steps"]:
        apply_ops(oix, st["ops"])
        op.set_state(*st["fleet"])
        res = []
        for reqs in st["batches"]:
            tokens, offsets, _ = ragged(reqs)
            idx, br, ma, _ = op.select_batch_tokens(tokens, offsets.astype(np.uint64)) if reqs else (np.zeros(0, np.int32),) * 3 + (0,)
            res.append((np.asarray(idx), np.asarray(br), np.asarray(ma)))
        out.append(res)
    return out


@pytest.mark.parametrize("jump", [64, 8])
def test_sequences_reach_the_slow_queue_and_every_branch(jump):
    """CPU guard of the GPU sequence tests below: the plan queues requests of every kind, shrinks right after a full queue, follows
    queued calls with imbalanced and no-healthy calls, reallocates lane 0's queue, has launches the tiled and streaming kernels take,
    and the oracle's answers cover every branch of the pick."""
    plan, want = build_plan(jump), run_oracle(jump)
    steps = plan["steps"]
    assert len(steps) >= 40
    kinds = {k for st in steps for ks in st["kinds"] for k in ks}
    assert {"multi_first", "multi_drain", "multi_last", "long", "b33"} <= kinds
    lens = [len(r) for st in steps for reqs in st["batches"] for r in reqs]
    nblks = {n // BS for n in lens}
    assert min(lens) < BS and {1, 32, 33} <= nblks and any(40 <= n <= MAX_BLOCKS for n in nblks) and max(nblks) <= MAX_BLOCKS
    if jump + 2 <= 32:
        assert any(jump + 1 < n <= 32 for n in nblks)   # one jump is not enough
    branches = [set(np.concatenate([r[1] for r in res]).tolist()) for res in want]
    assert {NO_HEALTHY, IMBALANCED, OVERLAP, MIN_LOAD} <= set().union(*branches)
    assert sum(int((r[1] == OVERLAP).sum()) for res in want for r in res) > 500

    def routed(i):   # the fleet lets the simple kernel reach the queue: some worker healthy, gate off
        return NO_HEALTHY not in branches[i] and IMBALANCED not in branches[i]

    lane0 = [i for i, st in enumerate(steps) if st["lane"] == 0]
    totals = {i: sum(len(b) for b in steps[i]["batches"]) for i in range(len(steps))}
    queued = {i: sum(queues(k, len(r) // BS, jump) for ks, reqs in zip(steps[i]["kinds"], steps[i]["batches"]) for k, r in zip(ks, reqs))
              for i in range(len(steps))}
    assert sum(1 for i in lane0 if routed(i) and queued[i]) >= 10
    full_queue = [i for i in lane0 if routed(i) and queued[i] == totals[i]]
    assert any(totals[b] < totals[a] for a, b in zip(lane0, lane0[1:]) if a in full_queue)   # a shrink right after a full queue
    first_q = min(i for i in lane0 if routed(i) and queued[i])
    assert any(branches[i] == {IMBALANCED} for i in lane0 if i > first_q)
    assert any(branches[i] == {NO_HEALTHY} for i in lane0 if i > first_q)
    # lane 0's queue is (re)allocated at 2.5 × (total + 2) + 64 words whenever a launch needs more than total + 2 words
    cap, allocs = 0, []
    for i in lane0:
        if totals[i] + 2 > cap:
            cap, allocs = 2.5 * (totals[i] + 2) + 64, allocs + [i]
    assert len(allocs) >= 3 and allocs[-1] < lane0[-1]   # the first allocation, then growth in the middle of the sequence
    assert len({st["lane"] for st in steps}) >= 3
    many = [st for st in steps if st["many"]]
    assert any(0 in [len(b) for b in st["batches"][1:-1]] and len({len(b) for b in st["batches"]}) > 1 for st in many)
    small = min(32, jump + 1) * BS
    fits = [st for st in steps if st["cap"] and all(len(r) // BS <= st["cap"] // BS for b in st["batches"] for r in b)]
    assert all(st["cap"] == small for st in fits)
    tile_ok = [st for st in fits if len({len(b) for b in st["batches"]}) == 1]     # uniform batches, max_blocks ≤ jump + 1 and ≤ 32
    assert len(tile_ok) >= 6 and len(fits) >= 8                                     # … the streaming kernel: max_blocks ≤ 32
    assert any(any(k.startswith("multi") for ks in st["kinds"] for k in ks) for st in tile_ok)
    assert any(op == "removed" for st in steps for op, _, _ in st["ops"]) and any(op == "stored" for st in steps for op, _, _ in st["ops"])


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------

class Device:
    """Device buffers of one call, freed together."""

    def __init__(self, pol):
        from smg_b200 import _lib
        self.h, self.L, self.ptrs = pol._h, _lib.load(), []

    def put(self, a):
        from smg_b200 import _lib
        a = np.ascontiguousarray(a)
        err = _lib.new_err()
        p = self.L.smgx_device_alloc(self.h.p, max(a.nbytes, 4), C.byref(err))
        assert p, "device allocation failed"
        self.ptrs.append(p)
        if a.nbytes:
            self.h.call("smgx_memcpy_h2d", p, a.ctypes.data_as(C.c_void_p), a.nbytes)
        return p

    def get(self, p, dtype, n):
        out = np.zeros(n, dtype)
        if n:
            self.h.call("smgx_memcpy_d2h", out.ctypes.data_as(C.c_void_p), p, out.nbytes)
        return out

    def free(self):
        for p in self.ptrs:
            self.L.smgx_device_free(self.h.p, p)
        self.ptrs = []


def poisoned_info(n):
    return np.full(max(n, 1) * INFO.itemsize, INFO_POISON, np.uint8).view(INFO)


def gpu_policy(urls, jump, max_tokens=MAX_BLOCKS * BS):
    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
    from smg_b200 import _lib
    assert C.sizeof(_lib.DecisionInfo) == INFO.itemsize
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **CFG), max_tokens_per_request=max_tokens)
    ws = [BasicWorker(u) for u in urls]
    pol.init_workers(ws)
    mon = pol.kv_event_monitor(BS)
    ix = mon.create_indexer("unknown", jump)
    pol.set_kv_event_monitor(mon)
    for i, u in enumerate(urls):
        assert ix.intern_worker(u) == i
    return pol, ws, ix


def set_fleet(pol, ws, fleet):
    loads, healthy, circuit = fleet
    for w, l, h, c in zip(ws, loads, healthy, circuit):
        w.set_load(int(l)); w.set_healthy(bool(h)); w.set_circuit_ok(bool(c))
    return pol._push_fleet(ws)


def launch_one(pol, dev, model, lane, reqs, cap):
    """Enqueue smgx_select_batch_tokens_device on `lane` with poisoned outputs; → a function that reads (picks, info, lengths) back."""
    tokens, offsets, lens = ragged(reqs)
    n = len(reqs)
    d_out, d_info = dev.put(np.full(n, POISON, np.int32)), dev.put(poisoned_info(n))
    pol._h.call("smgx_select_batch_tokens_device", model, lane, dev.put(tokens), dev.put(offsets), n, cap, d_out, d_info)
    return lambda: (dev.get(d_out, np.int32, n), dev.get(d_info, np.uint8, n * INFO.itemsize).view(INFO), lens)


def select_one(pol, model, lane, reqs, cap):
    dev = Device(pol)
    try:
        read = launch_one(pol, dev, model, lane, reqs, cap)
        pol._h.call("smgx_synchronize")
        return read()
    finally:
        dev.free()


def select_many(pol, model, batches, cap):
    """smgx_select_many_tokens_device (lane 0 for up to 32 batches) with poisoned outputs → [picks per batch]."""
    dev = Device(pol)
    try:
        nb = len(batches)
        tok, off, out, ns = [], [], [], []
        for reqs in batches:
            tokens, offsets, _ = ragged(reqs)
            tok.append(dev.put(tokens)); off.append(dev.put(offsets)); out.append(dev.put(np.full(max(len(reqs), 1), POISON, np.int32)))
            ns.append(len(reqs))
        pol._h.call("smgx_select_many_tokens_device", model, nb, (C.c_void_p * nb)(*tok), (C.c_void_p * nb)(*off), (C.c_uint32 * nb)(*ns), cap,
                    (C.c_void_p * nb)(*out))
        pol._h.call("smgx_synchronize")
        got = [dev.get(p, np.int32, max(n, 1)) for p, n in zip(out, ns)]
        for g, n in zip(got, ns):
            assert n or g[0] == POISON, "an empty batch had an output written"
        return [g[:n] for g, n in zip(got, ns)]
    finally:
        dev.free()


def check(tag, idx, info, lens, want):
    oidx, obr, oma = want
    assert not (idx == POISON).any(), f"{tag}: {(idx == POISON).sum()} picks never written"
    bad = np.nonzero(idx != oidx)[0]
    assert not bad.size, f"{tag}: {bad.size} of {idx.size} picks differ from the oracle, first request {bad[0]}: {idx[bad[0]]} vs {oidx[bad[0]]}"
    if info is not None:
        assert not (info["branch"] == INFO_POISON).any(), f"{tag}: decision info never written"
        assert np.array_equal(info["input"], lens), tag
        bad = np.nonzero(info["branch"] != obr)[0]
        assert not bad.size, f"{tag}: branch of request {bad[0]} is {info['branch'][bad[0]]}, the oracle's {obr[bad[0]]}"
        # matched = the overlap score of the event search.  On the imbalanced branch the oracle reports the approximate token tree's match,
        # which select_worker_min_load keeps up to date on the side (cache_aware.rs:378-400); the event-driven pick scores nothing there.
        ev = np.isin(obr, (OVERLAP, MIN_LOAD))
        got = info["matched"].astype(np.int64) * BS
        assert np.array_equal(got[ev], np.asarray(oma, np.int64)[ev]) and not got[~ev].any(), f"{tag}: matched lengths differ"


@pytest.mark.gpu
@pytest.mark.parametrize("jump", [64, 8])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_launch_sequence_matches_the_oracle(impl, jump):
    """The whole plan on one policy: every output written, every pick, branch and matched length equal to the oracle's, call after call."""
    plan, want = build_plan(jump), run_oracle(jump)
    with selected(impl):
        pol, ws, ix = gpu_policy(plan["urls"], jump)
        apply_ops(ix, plan["init"])
        for i, (st, exp) in enumerate(zip(plan["steps"], want)):
            apply_ops(ix, st["ops"])
            model = set_fleet(pol, ws, st["fleet"])
            tag = f"{impl}, jump {jump}, call {i} ({st['mix']}, lane {st['lane']}, n = {[len(b) for b in st['batches']]})"
            if st["many"]:
                for j, (got, e) in enumerate(zip(select_many(pol, model, st["batches"], st["cap"]), exp)):
                    check(f"{tag}, batch {j}", got, None, None, e)
            else:
                idx, info, lens = select_one(pol, model, st["lane"], st["batches"][0], st["cap"])
                check(tag, idx, info, lens, exp[0])


@pytest.mark.gpu
@pytest.mark.parametrize("d_fleet", ["imbalanced", "no_healthy"])
def test_queue_left_by_a_larger_launch_does_not_leak_into_later_ones(d_fleet):
    """Known answer for the slow queue's reset.  Four calls on lane 0, block size 16, jump 64, 4 workers:

      A  64 requests; request 0 is short, requests 1-63 have 40 blocks, so all 63 are queued (indices 1..63, never 0)
      B   8 short requests, none queued
      C   8 requests, 3 and 6 with 40 blocks: both queued
      D   8 short requests on an imbalanced fleet (or one with no healthy worker); 3 and 6 are full hits on a worker that is not the
          least loaded.  Every request gets the least-loaded worker with branch imbalanced_min_load (or -1 and no_healthy).

    With the exit counter at word total + 1 of the queue, as it was: A leaves its indices in words 1..63.  B's counter is word 9, which
    holds one of them, so B's last CTA never sees gridDim.x - 1 and the count and counter are not reset from then on.  C queues 3 and 6
    (count 2); D queues nothing but its slow kernel still reads count 2 and re-runs requests 3 and 6 of D with the event search, which
    overwrites their imbalanced (or no-healthy) picks with an overlap pick (or branch event_min_load).  All indices stay below 8 and every
    request fits max_blocks, so this is a wrong answer and not an out-of-bounds access."""
    W, jump = 4, 64
    urls = synth.worker_urls(W)
    with selected("simple"):
        pol, ws, ix = gpu_policy(urls, jump)
        op, oix = oracle_policy(urls, jump)
        seqs = synth.gen_sequences(8, 40 * BS, 7)
        rng = np.random.default_rng(7)
        ops = [("stored", 0, [(1 + k * 100 + i, h) for i, h in enumerate(orc.compute_request_content_hashes(seqs[k], BS))]) for k in range(8)]
        apply_ops(ix, ops); apply_ops(oix, ops)
        short = lambda: rng.integers(0, synth.VOCAB, size=int(rng.integers(1, 5)) * BS, dtype=np.uint32)   # noqa: E731
        balanced = (np.array([1, 2, 3, 4], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
        calls = [("A", [short()] + [seqs[k % 8].copy() for k in range(1, 64)], balanced),
                 ("B", [short() for _ in range(8)], balanced),
                 ("C", [seqs[k].copy() if k in (3, 6) else short() for k in range(8)], balanced)]
        d_reqs = [seqs[k][:4 * BS].copy() if k in (3, 6) else short() for k in range(8)]   # full hits on worker 0 (stored 40 blocks deep)
        if d_fleet == "imbalanced":
            calls.append(("D", d_reqs, (np.array([100, 0, 50, 80], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))))
        else:
            calls.append(("D", d_reqs, (balanced[0], np.zeros(W, np.uint8), np.ones(W, np.uint8))))
        for name, reqs, fleet in calls:
            model = set_fleet(pol, ws, fleet)
            op.set_state(*fleet)
            idx, info, lens = select_one(pol, model, 0, reqs, 0)
            tokens, offsets, _ = ragged(reqs)
            oidx, obr, oma, _ = op.select_batch_tokens(tokens, offsets.astype(np.uint64))
            check(f"call {name}", idx, info, lens, (np.asarray(oidx), np.asarray(obr), np.asarray(oma)))
        if d_fleet == "imbalanced":
            assert list(idx) == [1] * 8 and list(info["branch"]) == [IMBALANCED] * 8 and list(info["matched"]) == [0] * 8
        else:
            assert list(idx) == [-1] * 8 and list(info["branch"]) == [NO_HEALTHY] * 8
        assert list(obr[[3, 6]]) == list(info["branch"][[3, 6]])


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simple", "split"])
def test_request_over_the_cap_is_reported_once_and_does_not_leak(impl):
    """A request longer than max_request_tokens gets -1 and branch 255, and the next smgx_synchronize reports it once; the next call on
    the same lane, with another total and queued requests, is answered in full and synchronises cleanly."""
    from smg_b200 import SmgxError
    W, jump = 4, 8
    urls = synth.worker_urls(W)
    with selected(impl):
        pol, ws, ix = gpu_policy(urls, jump)
        op, oix = oracle_policy(urls, jump)
        seqs = synth.gen_sequences(12, 48 * BS, 11)
        ops = [("stored", k % W, [(1 + k * 100 + i, h) for i, h in enumerate(orc.compute_request_content_hashes(seqs[k], BS))]) for k in range(12)]
        apply_ops(ix, ops); apply_ops(oix, ops)
        fleet = (np.array([3, 1, 4, 1], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
        model = set_fleet(pol, ws, fleet)
        op.set_state(*fleet)
        # call 1: cap 32 blocks; request 5 has 40, requests of 12 and 20 blocks take more than one jump
        reqs = [seqs[k][:n * BS].copy() for k, n in enumerate([3, 12, 1, 20, 32, 40, 9, 2, 16, 5, 31, 7])]
        dev = Device(pol)
        try:
            read = launch_one(pol, dev, model, 0, reqs, 32 * BS)
            with pytest.raises(SmgxError, match="exceeded max_tokens_per_request"):
                pol._h.call("smgx_synchronize")
            pol._h.call("smgx_synchronize")   # reported once
            idx, info, lens = read()
        finally:
            dev.free()
        assert (idx[5], info["branch"][5]) == (-1, 255)
        tokens, offsets, _ = ragged(reqs)
        oidx, obr, oma, _ = op.select_batch_tokens(tokens, offsets.astype(np.uint64))
        keep = np.arange(len(reqs)) != 5
        check(f"{impl}, call 1", idx[keep], info[keep], lens[keep], (np.asarray(oidx)[keep], np.asarray(obr)[keep], np.asarray(oma)[keep]))
        # call 2, same lane: another total, the policy's own cap, requests of 40-48 blocks and several jumps
        reqs = [seqs[k % 12][:n * BS].copy() for k, n in enumerate([48, 2, 40, 13, 1, 33, 8, 45, 27, 3, 10, 41, 6, 30, 44, 9, 12, 19, 4, 47])]
        idx, info, lens = select_one(pol, model, 0, reqs, 0)
        tokens, offsets, _ = ragged(reqs)
        oidx, obr, oma, _ = op.select_batch_tokens(tokens, offsets.astype(np.uint64))
        check(f"{impl}, call 2", idx, info, lens, (np.asarray(oidx), np.asarray(obr), np.asarray(oma)))
