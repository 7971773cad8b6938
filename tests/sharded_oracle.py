"""Per-shard oracle of the worker-id-sharded event-driven pick (smg_b200/sharding.py).

Each rank indexes only its own contiguous range of the worker slice, runs the reference jump search (event_tree.rs:659-753) on that
shard's index alone, and emits its best eligible worker; smgx_shard_reduce_device merges the candidates in rank order.  This is what
the sharded pick computes, and it is NOT always the whole-fleet pick: the reference's count test (`count == active.len()`, :720), its
retain guard (`workers.len() < active.len()`, :611, :641) and the Single-entry shortcut (workers_if_single, no prefix check) decide
from the sizes of worker sets, and a shard only sees its own members of each set.  See DESIGN.md §4d for a counterexample.

The model here:
- one orc.PositionalIndexer per rank holding only that rank's workers, interned in local slice order;
- per request and per shard, the best eligible (healthy and circuit-ok) worker by (score, lower load, lower tree_size, higher slice
  index) — score_overlap's max_by_key with the last maximum (cache_aware.rs:806-818);
- the shards merged in rank order with the same last-max comparison;
- the prologue (no healthy worker, the f32 imbalance gate, the first min-load healthy worker) is global; it is taken from the
  whole-fleet orc.CacheAwarePolicy, asked about an empty request, so it is not restated here.

`matched` is the overlap score in blocks, as smgx_decision_info.matched reports it (the oracle policy reports tokens)."""
import numpy as np

from oracle import orc
from smg_b200.sharding import shard_range

NO_HEALTHY, IMBALANCED, OVERLAP, MIN_LOAD = 0, 1, 2, 3


class ShardedOracle:
    def __init__(self, urls, world, jump, cfg):
        self.urls, self.world, self.jump, self.bs = list(urls), world, jump, int(cfg["block_size"])
        n = len(self.urls)
        self.ranges = [shard_range(n, g, world) for g in range(world)]
        self.shards = []
        for lo, hi in self.ranges:
            ix = orc.PositionalIndexer(jump)
            for k, u in enumerate(self.urls[lo:hi]):
                assert ix.intern_worker(u) == k          # local ids follow local slice order
            self.shards.append(ix)
        self.policy = orc.CacheAwarePolicy(eviction_interval_secs=0, **cfg)
        self.policy.set_workers(self.urls)
        self.whole = orc.PositionalIndexer(jump)
        for u in self.urls:
            self.whole.intern_worker(u)
        self.policy.attach_indexer("unknown", self.whole)
        self.policy.set_kv_event_monitor(True)
        self.set_state(np.zeros(n, np.uint64), np.ones(n, np.uint8))

    def rank_of(self, g):
        return next(r for r, (lo, hi) in enumerate(self.ranges) if lo <= g < hi)

    def apply_stored(self, g, blocks):
        """Worker `g` (global slice index) stores `blocks` [(seq_hash, content_hash)] from position 0: its own shard and the whole fleet."""
        r = self.rank_of(g)
        self.shards[r].apply_stored(g - self.ranges[r][0], blocks)
        self.whole.apply_stored(g, blocks)

    def set_state(self, loads, healthy, circuit_ok=None):
        n = len(self.urls)
        self.loads = np.asarray(loads, np.uint64).copy()
        self.healthy = np.asarray(healthy, np.uint8).copy()
        self.circuit = np.ones(n, np.uint8) if circuit_ok is None else np.asarray(circuit_ok, np.uint8).copy()
        self.policy.set_state(self.loads, self.healthy, self.circuit)

    def prologue(self):
        """(branch, index) of the global prologue: NO_HEALTHY / IMBALANCED with their pick, or MIN_LOAD with the first min-load worker."""
        idx, br, _, _ = self.policy.select_batch_tokens(np.zeros(0, np.uint32), np.zeros(2, np.uint64))
        br = int(br[0])
        assert br in (NO_HEALTHY, IMBALANCED, MIN_LOAD), f"the whole-fleet oracle took branch {br} on an empty request (empty index?)"
        return br, int(idx[0])

    def candidate(self, rank, hashes):
        """The shard's best eligible worker for one request: (score, load, tree_size, global index), or None."""
        if not hashes:
            return None
        lo, hi = self.ranges[rank]
        scores, tsz = self.shards[rank].find_matches(hashes)
        best = None
        for k, s in sorted(scores.items()):                  # local slice order
            g = lo + k
            if s == 0 or not (self.healthy[g] and self.circuit[g]):
                continue
            c = (s, int(self.loads[g]), tsz[k], g)
            if best is None or _ge(c, best):
                best = c
        return best

    def select(self, tokens, offsets, max_blocks=None):
        """→ (idx int32[n], branch uint8[n], matched uint32[n]) of the sharded pick.  Requests of more than `max_blocks` blocks get no
        candidate from any shard (the candidate kernels flag them and store the empty candidate), so the merge picks the min-load worker."""
        tokens = np.asarray(tokens, np.uint32)
        offsets = np.asarray(offsets, np.int64)
        n = offsets.size - 1
        idx, br, ma = np.full(n, -1, np.int32), np.zeros(n, np.uint8), np.zeros(n, np.uint32)
        pbr, pidx = self.prologue()
        for i in range(n):
            if pbr != MIN_LOAD:
                idx[i], br[i] = pidx, pbr
                continue
            t = tokens[offsets[i]:offsets[i + 1]]
            best = None
            if max_blocks is None or t.size // self.bs <= max_blocks:
                hashes = orc.compute_request_content_hashes(t, self.bs)
                for g in range(self.world):
                    c = self.candidate(g, hashes)
                    if c is not None and (best is None or _ge(c, best)):
                        best = c
            if best is None:
                idx[i], br[i] = pidx, MIN_LOAD
            else:
                idx[i], br[i], ma[i] = best[3], OVERLAP, best[0]
        return idx, br, ma

    def select_whole(self, tokens, offsets):
        """The whole-fleet oracle's pick: (idx, branch, matched in blocks; 0 off the event branches)."""
        idx, br, ma, _ = self.policy.select_batch_tokens(np.asarray(tokens, np.uint32), np.asarray(offsets, np.uint64))
        ma = np.where((br == OVERLAP) | (br == MIN_LOAD), np.asarray(ma) // self.bs, 0).astype(np.uint32)
        return np.asarray(idx, np.int32), np.asarray(br, np.uint8), ma


def _ge(a, b):
    """a ≥ b under (score, Reverse(load), Reverse(tree_size)); a comes later in slice order, so equality lets it win (last max)."""
    return a[0] > b[0] or (a[0] == b[0] and (a[1] < b[1] or (a[1] == b[1] and a[2] <= b[2])))


# ---- indexes on which the sharded pick departs from the whole fleet ----------------------------------------------------------------

def _blocks(rng, n, bs):
    return [rng.integers(0, 50000, size=bs, dtype=np.uint32) for _ in range(n)]


def departure_case(kind, bs, world=2, seed=0):
    """A crafted index, fleet state and request on which the per-shard pick differs from the whole-fleet pick (jump 8, 9-block request).

    "count_test": A and D store c0..c7; C1 and C2 store x0..x7, c8 — the same content at position 8 under another prefix, a Single
      entry of size 2.  On the whole fleet the jump from 0 to 8 finds |{C1, C2}| = |{A, D}| and both score 9; D wins the tie (equal load
      and tree size, later index).  The shard {A, C1, C2} fails the count test, drains, and A keeps 9 (the drain's Single set is not
      smaller than {A}); the shard {D, …} has no entry at 8, so D scores 8.  Merged: A.
    "retain_guard": A and D store c0..c3; X1 and X2 store y0..y3, c4.  Both sides fail the count test.  On the whole fleet the drained
      position 4 holds the Single set {X1, X2}, not smaller than {A, D}, so nobody is dropped there and A, D both score 5; A has the lower
      load.  A's shard holds neither X, so A scores 4; D's shard holds both, so D keeps 5.  Merged: D.
    → dict(urls, world, stores {global index: [content hashes]}, loads, request tokens, whole, sharded) with the expected picks."""
    rng = np.random.default_rng(seed)
    req = _blocks(rng, 9, bs)
    other = _blocks(rng, 8, bs)
    c = orc.compute_request_content_hashes(np.concatenate(req), bs)
    x = orc.compute_request_content_hashes(np.concatenate(other), bs)
    if kind == "count_test":
        names = ["A", "C1", "C2", "D", "F"]                  # world 2: {A, C1, C2} | {D, F}
        stores = {"A": c[:8], "D": c[:8], "C1": x + [c[8]], "C2": x + [c[8]]}
        loads = {"A": 5, "D": 5}
        whole, sharded = "D", "A"
    elif kind == "retain_guard":
        names = ["A", "F1", "F2", "D", "X1", "X2"]           # world 2: {A, F1, F2} | {D, X1, X2}
        stores = {"A": c[:4], "D": c[:4], "X1": x[:4] + [c[4]], "X2": x[:4] + [c[4]]}
        loads = {"A": 3, "D": 7}
        whole, sharded = "A", "D"
    else:
        raise ValueError(kind)
    assert world == 2
    pos = {nm: i for i, nm in enumerate(names)}
    return dict(names=names, world=world, stores={pos[k]: v for k, v in stores.items()},
                loads=np.array([loads.get(nm, 6) for nm in names], np.uint64), tokens=np.concatenate(req).astype(np.uint32),
                whole=pos[whole], sharded=pos[sharded])


def seq_blocks(hashes, first_id):
    """[(seq_hash, content_hash)] for a chain stored from position 0, with fresh sequence ids."""
    return [(first_id + i, h) for i, h in enumerate(hashes)]


# ---- indexes built the way the sharded tests and bench.py's config-4 leg build them ---------------------------------------------------

def synth_stores(kind, n_workers, n_seq, T, bs, seed):
    """→ (sequences [n_seq, T], [(global worker, blocks)]).
    "replicas": each sequence stored by 1-5 random workers, each to a random depth (tests/test_gpu_sharded.py);
    "config4": sequence s stored whole by worker s mod n_workers (bench.py's sharded leg)."""
    from smg_b200 import synth
    seqs = synth.gen_sequences(n_seq, T, seed)
    rng = np.random.default_rng(seed)
    P, sid, out = T // bs, 1, []
    for s in range(n_seq):
        hs = orc.compute_request_content_hashes(seqs[s], bs)
        if kind == "replicas":
            for g in rng.choice(n_workers, size=min(n_workers, int(rng.integers(1, 6))), replace=False):
                depth = int(rng.integers(1, P + 1))
                out.append((int(g), seq_blocks(hs[:depth], sid)))
                sid += depth
        elif kind == "config4":
            out.append((s % n_workers, seq_blocks(hs, sid)))
            sid += P
        else:
            raise ValueError(kind)
    return seqs, out


def synth_requests(seqs, B, seed, bs, max_tokens):
    """Config-2 mix (full hits, stored prefixes + novel tokens, novel) at ragged lengths in [0, max_tokens] → (tokens, offsets u32)."""
    from smg_b200 import synth
    rng = np.random.default_rng(seed + 7)
    q = synth.gen_queries(seqs, B, seed, block=bs)
    lens = rng.integers(0, max_tokens + 1, size=B)
    lens[: B // 3] = min(max_tokens, q.shape[1])
    lens = np.minimum(lens, q.shape[1])
    offs = np.zeros(B + 1, np.uint32)
    np.cumsum(lens, out=offs[1:])
    tokens = np.concatenate([q[i, :lens[i]] for i in range(B)]).astype(np.uint32)
    return tokens, offs
