"""The event-driven pick on fleets wider than 64 workers, against the oracle.

Up to 64 interned workers a worker set is one u64 held in the slot.  Above 64 it is a row of `words` u64s: 2 words at 65-128
workers, 4 at 129-256, 8 at 257-512, 16 at 513-1024 and 32 at 1025-2048 (event_index.h, EventIndex::intern_worker).  Those fleets
run other kernels than the one-word ones: event_fused_kernel<false, …> on the default path, hash_blocks_kernel + event_search_warp_kernel
on the split path, warp_arg_best's reduction over the 32 lanes of a warp (one set word per lane), fleet_prepare_kernel's eligibility
words, and on the host EventIndex::rebuild (every set converted when the width grows) and the incremental flush (scatter_rows_kernel,
rows recycled through the free list).

Every scenario here is a list of operations (interning, index events, fleet states, picks) made from a seed alone.  play() runs one
on the oracle and, given a GPU policy, on the GPU as well, comparing pick, branch and matched length of every request with poisoned
outputs.  The CPU guard plays the same scenarios on the oracle alone and checks that they contain what the GPU tests rely on: winning
sets on both sides of the word boundaries and in lanes 16-31, ties decided between workers in different words, every branch, and
every kind of index change between picks.  The load-feedback stream and the two-rank sharded pick of test_gpu_feedback.py and
test_gpu_sharded.py run here at 2 and 32 set words."""
import functools

import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth

from . import test_gpu_feedback as feedback
from . import test_gpu_sharded as sharded
from .test_gpu_event_select import _oracle_policy
from .test_gpu_event_sequences import IMBALANCED, MIN_LOAD, NO_HEALTHY, OVERLAP, check, ragged, select_one, selected

MAX_BLOCKS = 64
CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5)
FLEETS = [64, 65, 128, 129, 1024, 1025, 2048]     # the first and last fleet size of each width from 1 to 32 words
BOUNDARIES = [64, 128, 1024]                      # ids b - 1 and b sit in different words; ids >= 1024 in lanes 16-31


# ---- scenarios (pure data, no GPU) ----------------------------------------------------------------------------------------------

class Builder:
    """Operations on one slice of workers:
      ("intern", url) ("refuse", url) ("stored", wid, blocks) ("removed", wid, seqs) ("cleared", wid) ("fleet", loads, healthy, circuit)
      ("pick", tag, reqs, extra) — extra: launches the index flush of this pick must cost over a repeat of it (None: not checked)."""

    def __init__(self, n_slice, bs, jump, seed):
        self.rng = np.random.default_rng(seed)
        self.bs, self.jump = bs, jump
        self.urls = synth.worker_urls(n_slice)
        self.ops, self.sid, self.kinds = [], 1, []
        self.seqs = synth.gen_sequences(400, MAX_BLOCKS * bs, 1000 + seed)
        self.next_seq = 0
        self.stored = []    # (seq index, depth): what requests can hit

    def seq(self):
        s = self.seqs[self.next_seq]
        self.next_seq += 1
        return s

    def intern(self, url):
        self.ops.append(("intern", url))

    def store(self, wid, tokens, depth, kind="stored"):
        """Blocks 0..depth-1 of `tokens` on worker `wid`; → the blocks (seq hash, content hash)."""
        hs = orc.compute_request_content_hashes(tokens[:depth * self.bs], self.bs)
        blocks = [(self.sid + i, hs[i]) for i in range(depth)]
        self.sid += depth
        self.ops.append(("stored", int(wid), blocks))
        self.kinds.append(kind)
        return blocks

    def remove(self, wid, blocks, kind="removed"):
        self.ops.append(("removed", int(wid), [b[0] for b in blocks]))
        self.kinds.append(kind)

    def fleet(self, loads, healthy=None, circuit=None):
        n = len(self.urls)
        self.ops.append(("fleet", np.asarray(loads, np.uint64), np.ones(n, np.uint8) if healthy is None else np.asarray(healthy, np.uint8),
                         np.ones(n, np.uint8) if circuit is None else np.asarray(circuit, np.uint8)))

    def noise(self, n):
        return self.rng.integers(0, synth.VOCAB, size=n, dtype=np.uint32)

    def requests(self, n, pool=None):
        """Requests of 0 blocks (empty and shorter than a block), 1 block, 2-31, exactly 32, 33-64 blocks, full hits of stored
        sequences, hits with a novel tail and novel ones; 30 % end in a partial block."""
        bs, rng = self.bs, self.rng
        pool = pool if pool is not None else self.stored
        out = []
        for i in range(n):
            k = i % 9
            s, depth = pool[int(rng.integers(0, len(pool)))]
            tokens = self.seqs[s]
            if k == 0:
                r = tokens[:int(rng.integers(0, bs))].copy()
            else:
                nb = {1: 1, 2: int(rng.integers(2, 32)), 3: 32, 4: int(rng.integers(33, MAX_BLOCKS + 1))}.get(k, depth)
                r = tokens[:nb * bs].copy()
                if k == 6 and nb > 1:
                    cut = int(rng.integers(1, nb))
                    r[cut * bs:] = self.noise((nb - cut) * bs)
                elif k == 7:
                    r = self.noise(nb * bs)
            if k and rng.random() < 0.3:
                r = np.concatenate([r, self.noise(int(rng.integers(1, bs)))])
            out.append(r)
        return out

    def pick(self, tag, reqs, extra=None):
        self.ops.append(("pick", tag, reqs, extra))


def shuffled_interning(b, n, seed):
    """Intern the first n slice URLs in a shuffled order, so that worker id != slice index.  → slice index of each id."""
    order = np.random.default_rng(seed).permutation(n)
    for k in order:
        b.intern(b.urls[k])
    return order


def multi_pair(b, ids_a, ids_b):
    """Two sequences sharing block 1 under different prefixes: a Multi entry at position 1 (as build_plan makes them)."""
    m, x = b.seq().copy(), b.seq().copy()
    bs = b.bs
    x[bs:2 * bs] = m[bs:2 * bs]
    s_m, s_x = b.next_seq - 2, b.next_seq - 1
    for w in ids_a:
        b.store(w, m, 8)
    for w in ids_b:
        b.store(w, x, 6, "multi")
    b.stored += [(s_m, 8), (s_x, 6)]


@functools.lru_cache(maxsize=None)
def matrix_plan(W, bs, jump):
    """A fleet of W interned workers, every width boundary below W held by tied winning sets."""
    b = Builder(W, bs, jump, W * 7 + bs + jump)
    rng = b.rng
    shuffled_interning(b, W, W + bs)
    pairs = [(x - 1, x) for x in BOUNDARIES if x < W] + ([(1024, W - 1), (1500, 2047)] if W > 1025 else [])
    if W <= 64:
        pairs = [(62, 63), (0, 63)]
    high = list(range(1024, W)) if W > 1024 else list(range(W // 2, W))
    for i in range(150):
        s = b.next_seq
        tokens = b.seq()
        if i % 3 == 0:                     # a boundary pair (and sometimes a third worker) at the same depth: tied scores
            ids = list(pairs[(i // 3) % len(pairs)])
            if rng.random() < 0.5:
                ids.append(int(rng.integers(0, W)))
            d = MAX_BLOCKS if rng.random() < 0.5 else int(rng.integers(1, MAX_BLOCKS + 1))
            depths = [d] * len(ids)
        else:
            n = int(rng.integers(1, 5))
            ids = [int(x) for x in rng.choice(high, size=min(n, len(high)), replace=False)] if i % 3 == 1 else \
                [int(x) for x in rng.choice(W, size=n, replace=False)]
            depths = [int(rng.integers(1, MAX_BLOCKS + 1)) for _ in ids]
        for w, d in zip(ids, depths):
            b.store(w, tokens, d)
        b.stored.append((s, max(depths)))
    for a, c in pairs:
        multi_pair(b, [a], [c])
    n = W
    loads = rng.integers(0, 3, size=n)                  # few load values: winning sets are decided by load and tree size
    healthy = (rng.random(n) > 0.05).astype(np.uint8)
    circuit = (rng.random(n) > 0.03).astype(np.uint8)
    b.fleet(loads, healthy, circuit)
    b.pick("balanced", b.requests(300))
    b.fleet(loads)
    b.pick("all healthy", b.requests(200))
    imb = loads.copy()
    imb[int(rng.integers(0, n))] = 300
    b.fleet(imb)
    b.pick("imbalanced", b.requests(40))
    b.fleet(loads, np.zeros(n, np.uint8))
    b.pick("no healthy", b.requests(20))
    return b


TIE_IDS = (5, 2047, 1100, 700)    # words 0, 31, 17 and 10, in the order the last-max rule picks them


@functools.lru_cache(maxsize=None)
def tie_plan(jump=8):
    """2048 workers; four of them (TIE_IDS) hold the same sequences to the same depth and nothing else, at equal loads, so every hit on
    those sequences is a tie decided by the slice index.  The highest slice index among them goes to id 5 (word 0), then 2047 (the last
    word), 1100 (lane 17) and 700 (word 10); each call takes the current winner out of the eligible set (health or circuit breaker)."""
    W, bs = 2048, 16
    b = Builder(W, bs, jump, 77)
    order = np.random.default_rng(78).permutation(W)
    top = sorted((order[i] for i in TIE_IDS), reverse=True)
    for i, sl in zip(TIE_IDS, top):
        order[i] = sl
    for k in order:
        b.intern(b.urls[k])
    rng = b.rng
    tie_pool = []
    for _ in range(12):
        s = b.next_seq
        tokens = b.seq()
        for w in TIE_IDS:
            b.store(w, tokens, 40)
        for w in rng.choice([x for x in range(W) if x not in TIE_IDS], size=3, replace=False):   # other workers, shallower
            b.store(int(w), tokens, int(rng.integers(1, 40)))
        tie_pool.append((s, 40))
    for _ in range(60):
        s = b.next_seq
        tokens = b.seq()
        d = int(rng.integers(1, MAX_BLOCKS + 1))
        for w in rng.choice([x for x in range(W) if x not in TIE_IDS], size=int(rng.integers(1, 4)), replace=False):
            b.store(int(w), tokens, d)
        b.stored.append((s, d))
    loads = rng.integers(3, 9, size=W)
    loads[[order[i] for i in TIE_IDS]] = 2
    healthy, circuit = np.ones(W, np.uint8), np.ones(W, np.uint8)

    def tie_requests():
        reqs = []
        for s, d in tie_pool:
            for n in (1, 17, 32, 33, 40):
                reqs.append(b.seqs[s][:n * bs].copy())
        return reqs + b.requests(40)

    for name, sl_off in [("word 0 wins", None), ("last word wins", ("h", 5)), ("lane 17 wins", ("c", 2047)),
                         ("word 10 wins", ("h", 1100)), ("word 0 again", "restore")]:
        if sl_off == "restore":
            healthy[:], circuit[:] = 1, 1
        elif sl_off is not None:
            (healthy if sl_off[0] == "h" else circuit)[order[sl_off[1]]] = 0
        b.fleet(loads, healthy.copy(), circuit.copy())
        b.pick(name, tie_requests())
    b.tie_slices = [int(order[i]) for i in TIE_IDS]
    return b


GROWTH = [60, 64, 65, 100, 128, 129, 256, 257, 512, 513, 1024, 1025, 1600, 2048]


@functools.lru_cache(maxsize=None)
def growth_plan(jump=8):
    """The slice is 2048 workers from the start; they are interned a few at a time, across every width boundary.  After each growth
    a pick runs before any new store (the answers come from rebuild's converted sets, Multi chains included); then stores on old and
    new ids, a removal and a clear, and another pick.  Last, a 2049th URL is refused and the index still answers."""
    W, bs = 2048, 16
    b = Builder(W, bs, jump, 31)
    rng = b.rng
    order = rng.permutation(W)
    loads = rng.integers(0, 6, size=W)
    b.fleet(loads)
    n = 0
    per_worker = {}
    for target in GROWTH:
        while n < target:
            b.intern(b.urls[order[n]])
            n += 1
        if target != GROWTH[0]:
            b.pick(f"{target} workers, converted sets", b.requests(120))
        top = [n - 1, n - 2] + ([64, 63] if n > 64 else []) + ([128, 127] if n > 128 else []) + ([1024, 1023] if n > 1024 else [])
        for i in range(10):          # stores on the newest ids and on both sides of each boundary below n, at equal depths
            s = b.next_seq
            tokens = b.seq()
            ids = {top[i % len(top)], top[(i + 1) % len(top)], int(rng.integers(0, n))}
            d = int(rng.integers(1, MAX_BLOCKS + 1))
            for w in ids:
                per_worker.setdefault(w, []).append(b.store(w, tokens, d))
            b.stored.append((s, d))
        multi_pair(b, [top[0], top[-1]], [top[1], int(rng.integers(0, n))])
        w = top[1]
        if per_worker.get(w):
            b.remove(w, per_worker[w].pop(0)[-2:])
        victim = int(rng.integers(0, n))
        b.ops.append(("cleared", victim))
        b.kinds.append("cleared")
        per_worker.pop(victim, None)
        b.pick(f"{target} workers, after new events", b.requests(120))
    b.ops.append(("refuse", synth.worker_urls(W + 1)[-1]))
    b.pick("after the refused intern", b.requests(120))
    return b


@functools.lru_cache(maxsize=None)
def churn_plan(W, jump=8):
    """W interned workers (shuffled), a small index, then 36 steps of one small event batch and one pick each.  The batches add a
    worker to an existing Single set, make new entries, upgrade Single entries to Multi at position 1, empty Single sets (row freed,
    slot a tombstone) and Multi nodes, reuse freed rows, clear workers, and grow the table past one rebuild.  Two steps are checked for
    the launches of the incremental flush: a store that only dirties a row (1 launch) and a new entry on a recycled row (2)."""
    bs = 16
    b = Builder(W, bs, jump, 1000 + W)
    rng = b.rng
    shuffled_interning(b, W, W + 5)
    far = [0, 63, 64, W - 1] + ([1024, 1500] if W > 1024 else [127, 128])
    solo, shared = [], []      # (wid, blocks) stored by one worker only / (seq, depth, blocks) that others may join
    for i in range(60):
        s = b.next_seq
        tokens = b.seq()
        w = far[i % len(far)] if i % 2 else int(rng.integers(0, W))
        d = int(rng.integers(2, 9))
        blocks = b.store(w, tokens, d)
        (solo if i % 3 == 0 else shared).append((w, blocks) if i % 3 == 0 else (s, d, w))
        b.stored.append((s, d))
    b.fleet(rng.integers(0, 4, size=W))
    b.pick("initial", b.requests(60))

    def new_entries(nseq, depth_max):
        for _ in range(nseq):
            s = b.next_seq
            tokens = b.seq()
            w = far[int(rng.integers(0, len(far)))] if rng.random() < 0.5 else int(rng.integers(0, W))
            d = int(rng.integers(1, depth_max + 1))
            blocks = b.store(w, tokens, d, "new")
            b.stored.append((s, d))
            if rng.random() < 0.5:
                solo.append((w, blocks))
            else:
                shared.append((s, d, w))

    for step in range(36):
        kind = ["join", "empty", "reuse", "multi", "grow", "cleared"][step % 6]
        extra = None
        if kind == "join":           # the same blocks on another worker: same prefixes, only the set's row changes
            s, d, w0 = shared[int(rng.integers(0, len(shared)))]
            w = int(rng.choice([x for x in far if x != w0]))
            b.store(w, b.seqs[s], d, "join")
            extra = 1 if step < 5 else None     # before the first clear: the set still exists, the step dirties its row alone
        elif kind == "empty":        # the only worker of Single sets leaves: rows freed, slots become tombstones
            w, blocks = solo.pop(int(rng.integers(0, len(solo))))
            b.remove(w, blocks, "empty")
        elif kind == "reuse":        # one new entry: a slot and a recycled row
            s = b.next_seq
            tokens = b.seq()
            w = far[step % len(far)]
            solo.append((w, b.store(w, tokens, 1, "reuse")))
            b.stored.append((s, 1))
            extra = 2 if step < 5 else None     # far from the table's growth threshold: no rebuild, no full upload
        elif kind == "multi":        # Single → Multi at position 1, and a Multi node emptied again on every other such step
            m_s, m_d, m_w = shared[int(rng.integers(0, len(shared)))]
            x = b.seq().copy()
            x[bs:2 * bs] = b.seqs[m_s][bs:2 * bs]
            w = far[(step // 6) % len(far)]
            if m_d >= 2:
                blocks = b.store(w, x, 4, "multi")
                b.stored.append((b.next_seq - 1, 4))
                if step % 12 == 9:
                    b.remove(w, blocks[1:2], "multi_removed")
            else:
                new_entries(1, 8)
        elif kind == "grow":         # ≤ 60 entries: a slot and a row each, fewer dirty records than 1024 slots / 8
            new_entries(10, 6)
        else:
            w = int(rng.integers(0, W))
            b.ops.append(("cleared", w))
            b.kinds.append("cleared")
            solo[:] = [(x, bl) for x, bl in solo if x != w]
            new_entries(4, 5)
        b.pick(f"step {step} ({kind})", b.requests(60), extra)
    return b


@functools.lru_cache(maxsize=None)
def wide_slice_plan(jump=8):
    """A slice of 2100 workers with 2048 interned; the 52 others (id -1) can only be picked by min-load.  Equal loads everywhere, so
    the first-minimum rule of fleet_prepare_kernel's strided reduction decides min_load_idx; then the imbalance gate and no healthy worker."""
    W, n_slice, bs = 2048, 2100, 16
    b = Builder(n_slice, bs, jump, 5)
    rng = b.rng
    outside = {300, 301, 555, 1777, 2099} | set(int(x) for x in rng.choice(n_slice, size=47, replace=False))
    while len(outside) < 52:
        outside.add(int(rng.integers(0, n_slice)))
    inside = [i for i in rng.permutation(n_slice) if i not in outside][:W]
    assert len(inside) == W and len(set(inside)) == W
    for k in inside:
        b.intern(b.urls[k])
    for _ in range(80):
        s = b.next_seq
        tokens = b.seq()
        d = int(rng.integers(1, MAX_BLOCKS + 1))
        for w in rng.choice(W, size=int(rng.integers(1, 4)), replace=False):
            b.store(int(w), tokens, d)
        b.stored.append((s, d))
    healthy = np.ones(n_slice, np.uint8)
    healthy[:300] = 0
    loads = np.full(n_slice, 5, np.uint64)
    b.fleet(loads, healthy)
    b.pick("equal loads, first healthy is not interned", b.requests(100))
    loads2 = loads.copy()
    loads2[[2099, 1999, 1200, 777, 555]] = 1       # the first minimum is 555 (not interned), in another thread's stride than 777 …
    b.fleet(loads2, healthy)
    b.pick("equal minima in several strides", b.requests(100))
    healthy2 = healthy.copy()
    healthy2[555] = 0                               # … then 777 (interned)
    b.fleet(loads2, healthy2)
    b.pick("first minimum interned", b.requests(100))
    imb = loads2.copy()
    imb[10] = 1000
    b.fleet(imb, healthy2)
    b.pick("imbalanced", b.requests(30))
    b.fleet(loads2, np.zeros(n_slice, np.uint8))
    b.pick("no healthy", b.requests(20))
    return b


# ---- playing a scenario --------------------------------------------------------------------------------------------------------

class Gpu:
    """The GPU side of play(): a policy over the same slice, interning in the same order."""

    def __init__(self, b, feedback=False):
        from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
        self.pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, block_size=b.bs, **CFG), max_batch=8192,
                                    max_tokens_per_request=(MAX_BLOCKS + 1) * b.bs)
        self.ws = [BasicWorker(u) for u in b.urls]
        self.pol.init_workers(self.ws)
        mon = self.pol.kv_event_monitor(b.bs)
        self.ix = mon.create_indexer("unknown", b.jump)
        self.pol.set_kv_event_monitor(mon)
        self.feedback = feedback
        if feedback:
            self.pol.set_load_feedback(True)


def play(b, gpu=None):
    """Run the scenario on the oracle (and on `gpu`, comparing every pick).  → per pick: (tag, reqs, (picks, branches, matched tokens),
    winning sets, the oracle's entry count)."""
    from smg_b200 import SmgxError
    bs = b.bs
    op, oix = _oracle_policy(b.urls, dict(block_size=bs, **CFG), b.jump, bs)
    fleet = None
    out = []
    model = None
    for o in b.ops:
        kind = o[0]
        if kind == "intern":
            wid = oix.intern_worker(o[1])
            if gpu:
                assert gpu.ix.intern_worker(o[1]) == wid
            continue
        if kind == "refuse":
            if gpu:
                with pytest.raises(SmgxError, match="MAX_WORKERS"):
                    gpu.ix.intern_worker(o[1])
                assert gpu.ix.worker_id(o[1]) is None
            continue
        if kind == "stored":
            oix.apply_stored(o[1], o[2])
        elif kind == "removed":
            oix.apply_removed(o[1], o[2])
        elif kind == "cleared":
            oix.apply_cleared(o[1])
        if kind in ("stored", "removed", "cleared"):
            if gpu:
                getattr(gpu.ix, "apply_" + kind)(*o[1:])
            continue
        if kind == "fleet":
            fleet = o[1:]
            op.set_state(*fleet)
            if gpu:
                for w, l, h, c in zip(gpu.ws, *fleet):
                    w.set_load(int(l)); w.set_healthy(bool(h)); w.set_circuit_ok(bool(c))
                model = gpu.model = gpu.pol._push_fleet(gpu.ws)
            continue
        _, tag, reqs, extra = o
        tokens, offsets, lens = ragged(reqs)
        if gpu and gpu.feedback:
            want = op.select_batch_tokens_feedback(tokens, offsets.astype(np.uint64))[:3]
        else:
            want = op.select_batch_tokens(tokens, offsets.astype(np.uint64))[:3]
        want = tuple(np.asarray(x) for x in want)
        out.append((tag, reqs, want, winsets(b, oix, reqs, fleet), oix.entry_count()))
        if gpu and gpu.feedback:
            idx, info = gpu.pol.select_worker_batch(gpu.ws, tokens=tokens, offsets=offsets)
            assert np.array_equal(idx, want[0]), f"{tag}: {(idx != want[0]).sum()} picks differ"
            assert [i.branch for i in info] == list(want[1]), tag
            assert [i.matched * bs if i.branch == OVERLAP else i.matched for i in info] == list(want[2]), tag
        elif gpu:
            before = gpu.pol.kernel_launches()
            idx, info, got_lens = select_one(gpu.pol, model, 0, reqs, 0)
            first = gpu.pol.kernel_launches() - before
            # check() reads matched lengths in blocks of 16 tokens
            ev = np.isin(want[1], (OVERLAP, MIN_LOAD))
            check(tag, idx, info, got_lens, (want[0], want[1], np.where(ev, want[2] // bs * 16, want[2])))
            if extra is not None:
                before = gpu.pol.kernel_launches()
                idx2, _, _ = select_one(gpu.pol, model, 0, reqs, 0)
                assert np.array_equal(idx2, idx), tag
                assert first - (gpu.pol.kernel_launches() - before) == extra, \
                    f"{tag}: the index flush cost {first - (gpu.pol.kernel_launches() - before)} launches, expected {extra}"
    return out


def winsets(b, oix, reqs, fleet):
    """Per request, the eligible interned workers with the best overlap score (the kernel's winning set), by worker id."""
    loads, healthy, circuit = fleet
    ok = {}
    for i, u in enumerate(b.urls):
        wid = oix.worker_id(u)
        if wid is not None and healthy[i] and circuit[i]:
            ok[wid] = i
    out = []
    for r in reqs:
        nb = len(r) // b.bs
        if nb == 0:
            out.append(set())
            continue
        sc, _ = oix.find_matches(orc.compute_request_content_hashes(r[:nb * b.bs], b.bs))
        sc = {w: s for w, s in sc.items() if w in ok and s > 0}
        best = max(sc.values(), default=0)
        out.append({w for w, s in sc.items() if s == best} if best else set())
    return out


# ---- CPU guards ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("W", FLEETS)
def test_width_matrix_reaches_every_word_boundary_and_branch(W):
    """Guard of test_width_matrix_matches_the_oracle, on the oracle alone: winning sets hold both ids of each word boundary below W,
    span several words and reach lanes 16-31 (ids >= 1024), and every branch of the pick occurs."""
    res = play(matrix_plan(W, 16, 8))
    sets = [s for _, _, _, ws, _ in res for s in ws]
    for x in BOUNDARIES:
        if x < W:
            assert sum(1 for s in sets if x - 1 in s and x in s) >= 5, f"no winning set holds {x - 1} and {x}"
    if W > 64:
        assert sum(1 for s in sets if len({w >> 6 for w in s}) > 1) >= 100
    if W > 1024:
        assert sum(1 for s in sets if any(w >= 1024 for w in s)) >= 50 and any(W - 1 in s for s in sets)
    br = np.concatenate([w[1] for _, _, w, _, _ in res])
    assert {NO_HEALTHY, IMBALANCED, OVERLAP, MIN_LOAD} <= set(br.tolist())
    assert (br == OVERLAP).sum() > 200


def test_tie_growth_and_churn_scenarios_contain_what_the_gpu_tests_rely_on():
    """Guard of the tie, growth and churn tests, on the oracle alone: ties between TIE_IDS are decided across words and each call's
    winner is the one the test names; the churn scenarios contain every kind of index change and grow the table past a rebuild while
    wide (the table starts at 1024 slots and grows when half full); the growth scenario removes, clears and ends with a refused intern."""
    t = tie_plan()
    tres = play(t)
    n_tie = sum(1 for *_, ws, _ in tres for s in ws if len({w >> 6 for w in s & set(TIE_IDS)}) > 1)
    assert n_tie >= 200
    assert [int(r[2][0][0]) for r in tres] == [t.tie_slices[k] for k in (0, 1, 2, 3, 0)]   # request 0 of each call: a tie hit
    for W in (129, 2048):
        c = churn_plan(W)
        assert {"join", "empty", "reuse", "multi", "multi_removed", "new", "cleared"} <= set(c.kinds)
        assert sum(1 for o in c.ops if o[0] == "pick") >= 31
        assert sorted(o[3] for o in c.ops if o[0] == "pick" and o[3] is not None) == [1, 2]
        entries = [e for *_, e in play(c)]
        assert entries[0] < 400 and max(entries) > 520
    g = growth_plan()
    assert {"stored", "multi", "removed", "cleared"} <= set(g.kinds)
    assert g.ops[-2][0] == "refuse" and g.ops[-1][0] == "pick"


def test_host_mirror_interns_2048_workers_and_refuses_the_next():
    """The host side of the index on a policy without a device (device_id = -1): the growth scenario's events keep entry_count and
    current_size equal to the oracle's through every width growth; 2048 interns succeed and the 2049th is refused."""
    from smg_b200 import PositionalIndexer, SmgxError, _lib
    b = growth_plan()
    ix = PositionalIndexer.standalone(b.jump, device_id=-1)
    oix = orc.PositionalIndexer(b.jump)
    n_checks = 0
    for o in b.ops:
        if o[0] == "intern":
            assert ix.intern_worker(o[1]) == oix.intern_worker(o[1])
        elif o[0] in ("stored", "removed", "cleared"):
            getattr(ix, "apply_" + o[0])(*o[1:])
            getattr(oix, "apply_" + o[0])(*o[1:])
        elif o[0] == "pick":
            assert (ix.entry_count(), ix.current_size()) == (oix.entry_count(), oix.current_size()), o[1]
            n_checks += 1
        elif o[0] == "refuse":
            with pytest.raises(SmgxError) as e:
                ix.intern_worker(o[1])
            assert e.value.code == _lib.INVALID_ARGUMENT and "MAX_WORKERS" in str(e.value)
            assert ix.worker_id(o[1]) is None
    assert n_checks == 2 * len(GROWTH)
    assert ix.worker_id(b.urls[0]) is not None and ix.entry_count() == oix.entry_count() > 0


# ---- GPU -------------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("bs,jump", [(16, 64), (16, 8), (4, 64), (4, 8)])
@pytest.mark.parametrize("impl", ["simple", "split"])
@pytest.mark.parametrize("W", FLEETS)
def test_width_matrix_matches_the_oracle(W, impl, bs, jump):
    """Every width from 1 to 32 words at its first and last fleet size, on the default kernel family (event_fused_kernel<false, …>
    above 64 workers) and the split one (hash_blocks_kernel + event_search_warp_kernel): bit-exact picks, and the family reached."""
    b = matrix_plan(W, bs, jump)
    with selected(impl):
        g = Gpu(b)
        play(b, g)
        reqs = b.requests(50)
        select_one(g.pol, g.model, 0, reqs, 0)
        before = g.pol.kernel_launches()
        select_one(g.pol, g.model, 0, reqs, 0)
        n = g.pol.kernel_launches() - before
    if impl == "split":
        assert n == 2, f"hash + search: {n} launches"
    elif W > 64:
        assert n == 1, f"event_fused_kernel: {n} launches"


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simple", "split", "feedback"])
def test_ties_across_words_follow_the_slice_index(impl):
    """Four workers in words 0, 31, 17 and 10 tie on score, load and tree size; the highest eligible slice index wins, and taking the
    winner out of the eligible set (health, then circuit breaker) hands the pick to the next across a word boundary."""
    b = tie_plan()
    with selected("simple" if impl == "feedback" else impl):
        play(b, Gpu(b, feedback=impl == "feedback"))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simple", "split"])
def test_width_growth_after_entries_exist(impl):
    """Interning across every width boundary with a populated index: picks on converted sets, then on new events; the 2049th URL is
    refused with MAX_WORKERS, stays unknown, and the next pick still equals the oracle."""
    b = growth_plan()
    with selected(impl):
        play(b, Gpu(b))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simple", "split"])
@pytest.mark.parametrize("W", [129, 2048])
def test_index_churn_between_picks(W, impl):
    """One small event batch and one pick per step: joins, new entries, Single → Multi, emptied sets and Multi nodes, recycled rows,
    clears and a table rebuild, each reaching the device through the incremental flush."""
    b = churn_plan(W)
    with selected(impl):
        play(b, Gpu(b))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simple", "split"])
def test_slice_wider_than_the_index(impl):
    """2100 slice entries over 2048 interned workers: min-load picks of entries the index does not know, the first minimum among equal
    loads in different strides of fleet_prepare_kernel, the imbalance gate and no healthy worker."""
    b = wide_slice_plan()
    with selected(impl):
        play(b, Gpu(b))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simple", "split"])
def test_shard_candidates_of_one_rank_match_the_oracle(impl):
    """The candidate mode of both kernel families at 2048 workers (32 words), through a one-rank ShardedEventRouter."""
    from smg_b200 import CacheAwareConfig
    from smg_b200.sharding import ShardedEventRouter
    b = matrix_plan(2048, 16, 8)
    with selected(impl):
        router = ShardedEventRouter(b.urls, 0, 1, CacheAwareConfig(eviction_interval_secs=0, block_size=16, **CFG), jump_size=b.jump,
                                    max_tokens_per_request=MAX_BLOCKS * 16)
        op, oix = _oracle_policy(b.urls, dict(block_size=16, **CFG), b.jump, 16)
        for u in b.urls:
            oix.intern_worker(u)
        # the router interns in slice order: replay the plan's events under those ids
        remap = {}
        for o in b.ops:
            if o[0] == "intern":
                remap[len(remap)] = b.urls.index(o[1])
        for o in b.ops:
            if o[0] == "stored":
                router.indexer.apply_stored(remap[o[1]], o[2]); oix.apply_stored(remap[o[1]], o[2])
        fleets = [o[1:] for o in b.ops if o[0] == "fleet"][:2]
        for k, (loads, healthy, circuit) in enumerate(fleets):
            router.set_fleet_state(loads, healthy, circuit)
            op.set_state(loads, healthy, circuit)
            reqs = b.requests(300)
            tokens, offsets, _ = ragged(reqs)
            got = router.select(tokens, offsets, MAX_BLOCKS * 16, lambda a: a)
            want = np.asarray(op.select_batch_tokens(tokens, offsets.astype(np.uint64))[0])
            assert np.array_equal(got, want), f"fleet {k}: {(got != want).sum()} picks differ"


@pytest.mark.gpu
@pytest.mark.parametrize("n_workers,seed", [(1025, 4), (2048, 5)])
def test_feedback_stream_at_32_words(n_workers, seed):
    """test_gpu_feedback's request stream at 32 set words: the fused kernel writes every word of each request's tied set and
    feedback_resolve_kernel walks them, with 2048 loads in shared memory.  Round 2 starts the imbalance gate at 68 over a fleet at 3:
    it closes after one min-load pick per worker (at 80, as the 64-worker test has it, it would take ≈ 13 × n_workers > B picks)."""
    T, bs, B = 512, 16, 4096
    pol, ws, op, seqs, rng = feedback._setup(n_workers, T, bs, 64, seed)
    pol.set_load_feedback(True)
    q = synth.gen_queries(seqs, B, seed, block=bs)
    novel = rng.random(B) < 0.3
    q[novel] = rng.integers(0, 50000, size=(int(novel.sum()), T), dtype=np.uint32)
    tokens, offsets = synth.ragged(q)
    for rnd in range(3):
        loads = synth.poisson_loads(n_workers, 8, seed + rnd)
        healthy = (rng.random(n_workers) > 0.1).astype(np.uint8)
        if rnd == 2:
            loads[:] = 3
            healthy[:] = 1
            loads[5] = 68
        for i, w in enumerate(ws):
            w.set_load(int(loads[i])); w.set_healthy(bool(healthy[i]))
        op.set_state(loads, healthy, [1] * n_workers)
        idx, info = pol.select_worker_batch(ws, tokens=tokens, offsets=offsets)
        oidx, obr, oma, _ = op.select_batch_tokens_feedback(tokens, offsets.astype(np.uint64))
        assert np.array_equal(idx, oidx), f"round {rnd}: {(idx != oidx).sum()} picks differ"
        assert [i.branch for i in info] == list(obr)
        assert [i.matched * bs if i.branch == OVERLAP else i.matched for i in info] == list(oma)
        minload = np.isin(np.asarray(obr), (IMBALANCED, MIN_LOAD))
        assert minload.sum() > B // 10 and len(set(int(x) for x in oidx[minload])) > 8
        if rnd == 2:
            assert (np.asarray(obr) == IMBALANCED).sum() > 100 and (np.asarray(obr) == OVERLAP).sum() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("world,n_workers,seed", [(2, 130, 5),     # 65 workers per shard: 2 set words
                                                   (2, 4096, 6)])   # 2048 workers per shard: 32 set words
def test_sharded_pick_at_2_and_32_words_per_shard(world, n_workers, seed):
    """test_gpu_sharded's two-rank pick (gloo and peer-memory exchange) with shards of 2 and of 32 set words."""
    sharded.test_sharded_pick_matches_oracle_on_whole_fleet(world, n_workers, seed)
