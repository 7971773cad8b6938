"""The worker-id-sharded pick, candidates and merge, in ONE process: `world` ranks of a fleet on cuda:0, each a CacheAwarePolicy built the
way ShardedEventRouter builds it, smgx_shard_candidates_device on every rank into a [world][n] candidate array and a [world] summary
array, then smgx_shard_reduce_device — against the per-shard oracle (tests/sharded_oracle.py): picks, branches and matched scores.

No collective, no peer memory and no spawned process, so the cases are cheap: ties on rank boundaries, the global prologue re-derived
from the shards' summaries (equal minima on two ranks, minima and maxima on unhealthy or circuit-open workers, all-unhealthy and empty
ranks, no healthy worker, the f32 gate above 2^24), every candidate site (fleets of 1 to 2048 workers per shard, block size 16 and
others, 0-token, sub-block, 32-block fast-path, longer, drained and Multi-entry requests, batches of 1 to 5000), the indexes on which the
shards depart from the whole fleet, and requests longer than max_tokens_per_request.

The merge reports `input` = 0 in smgx_decision_info: it only sees candidates, not the requests' lengths."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth
from tests.sharded_oracle import (IMBALANCED, MIN_LOAD, NO_HEALTHY, OVERLAP, ShardedOracle, departure_case, seq_blocks, synth_requests,
                                  synth_stores)
from tests.test_gpu_event_sequences import selected

pytestmark = pytest.mark.gpu

CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5)
CAND = np.dtype([("score", "<u4"), ("local_idx", "<u4"), ("load", "<u8"), ("tree_size", "<u8")])
FLEET = np.dtype([("min_load_idx", "<i4"), ("first_healthy", "<i4"), ("n_healthy", "<u4"), ("imbalanced", "<u4"), ("min_load", "<u8"),
                  ("max_load", "<u8"), ("min_healthy_load", "<u8")])
INFO = np.dtype([("matched", "<u4"), ("input", "<u4"), ("branch", "u1"), ("nodes", "u1"), ("reserved", "u1", 2)])
POISON, INFO_POISON = -7, 0xA5
assert CAND.itemsize == 24 and FLEET.itemsize == 40 and INFO.itemsize == 12


class Fleet:
    """One sharded fleet: the GPU ranks (all on cuda:0) and the per-shard oracle beside them."""

    def __init__(self, urls, world, bs, jump, max_tokens, cfg=CFG):
        from smg_b200 import CacheAwareConfig
        from smg_b200.sharding import ShardedEventRouter
        self.urls, self.world, self.bs, self.T = list(urls), world, bs, max_tokens
        conf = CacheAwareConfig(eviction_interval_secs=0, block_size=bs, **cfg)
        self.routers = [ShardedEventRouter(self.urls, g, world, conf, jump_size=jump, device_id=0, max_batch=8192, max_tokens_per_request=max_tokens)
                        for g in range(world)]
        self.oracle = ShardedOracle(self.urls, world, jump, dict(cfg, block_size=bs))
        self.sid = 1
        self.set_state(np.full(len(self.urls), 4, np.uint64), np.ones(len(self.urls), np.uint8))

    def close(self):
        for r in self.routers:
            r.policy.close()

    def store(self, g, hashes):
        """Worker g (global index) stores the chain `hashes` from position 0."""
        blocks = seq_blocks(hashes, self.sid)
        self.sid += len(hashes) + 1
        rt = self.routers[self.oracle.rank_of(g)]
        rt.indexer.apply_stored(rt.local_id(g), blocks)
        self.oracle.apply_stored(g, blocks)

    def set_state(self, loads, healthy, circuit=None):
        for rt in self.routers:
            rt.set_fleet_state(loads, healthy, circuit)
        self.oracle.set_state(loads, healthy, circuit)

    def run(self, tokens, offsets):
        """→ (picks, info, candidates [world][n], summaries [world], status of each rank's smgx_synchronize after its candidates)."""
        from smg_b200 import _lib
        tokens, offsets = np.ascontiguousarray(tokens, np.uint32), np.ascontiguousarray(offsets, np.uint32)
        n, W = offsets.size - 1, self.world
        h0, L = self.routers[0].policy._h, _lib.load()
        err = _lib.new_err()
        bufs = []

        def alloc(nbytes, host=None):
            d = L.smgx_device_alloc(h0.p, max(nbytes, 16), C.byref(err))
            assert d, "device allocation failed"
            bufs.append(d)
            if host is not None and host.nbytes:
                h0.call("smgx_memcpy_h2d", C.c_void_p(d), host.ctypes.data_as(C.c_void_p), host.nbytes)
            return d
        try:
            d_tok, d_off = alloc(tokens.nbytes, tokens), alloc(offsets.nbytes, offsets)
            d_cand = alloc(W * n * CAND.itemsize, np.full(W * n * CAND.itemsize, 0xCD, np.uint8))
            d_fleet = alloc(W * FLEET.itemsize, np.full(W * FLEET.itemsize, 0xCD, np.uint8))
            d_out = alloc(n * 4, np.full(max(n, 1), POISON, np.int32))
            d_info = alloc(n * INFO.itemsize, np.full(max(n, 1) * INFO.itemsize, INFO_POISON, np.uint8))
            for g, rt in enumerate(self.routers):
                rt.policy._h.call("smgx_shard_candidates_device", rt.model, 0, C.c_void_p(d_tok), C.c_void_p(d_off), n, self.T,
                                  C.c_void_p(d_cand + g * n * CAND.itemsize), C.c_void_p(d_fleet + g * FLEET.itemsize))
            status = []
            for rt in self.routers:
                try:
                    rt.policy._h.call("smgx_synchronize")
                    status.append(_lib.SUCCESS)
                except _lib.SmgxError as e:
                    status.append(e.code)
            gbase = self.routers[0].gbase
            h0.call("smgx_shard_reduce_device", 0, C.c_void_p(d_cand), C.c_void_p(d_fleet), gbase.ctypes.data_as(C.c_void_p), W, n,
                    C.c_void_p(d_out), C.c_void_p(d_info))
            h0.call("smgx_synchronize")
            out = np.zeros(max(n, 1), np.int32)
            info = np.zeros(max(n, 1), INFO)
            cand = np.zeros(max(W * n, 1), CAND)
            fleet = np.zeros(W, FLEET)
            for host, d, nbytes in ((out, d_out, n * 4), (info, d_info, n * INFO.itemsize), (cand, d_cand, W * n * CAND.itemsize),
                                    (fleet, d_fleet, W * FLEET.itemsize)):
                if nbytes:
                    h0.call("smgx_memcpy_d2h", host.ctypes.data_as(C.c_void_p), C.c_void_p(d), nbytes)
            return out[:n], info[:n], cand[:W * n].reshape(W, n), fleet, status
        finally:
            for d in bufs:
                L.smgx_device_free(h0.p, C.c_void_p(d))

    def check(self, tokens, offsets, tag="", max_blocks=None):
        """Run on the GPU, compare with the per-shard oracle; → (picks, branches) for further assertions."""
        from smg_b200 import _lib
        idx, info, cand, fleet, status = self.run(tokens, offsets)
        want_i, want_b, want_m = self.oracle.select(tokens, offsets, max_blocks)
        assert status == [_lib.SUCCESS] * self.world, (tag, status)
        bad = np.nonzero((idx != want_i) | (info["branch"] != want_b) | (info["matched"] != want_m))[0]
        assert bad.size == 0, (tag, [(int(i), int(idx[i]), int(want_i[i]), int(info["branch"][i]), int(want_b[i]), int(info["matched"][i]),
                                      int(want_m[i])) for i in bad[:8]])
        assert not info["input"].any() and not info["nodes"].any(), tag     # the merge never sees the requests' lengths
        self.check_summaries(fleet, tag)
        return idx, info["branch"]

    def check_summaries(self, fleet, tag):
        """Each rank's 40 B summary against its own slice of the fleet state."""
        o = self.oracle
        for g, (lo, hi) in enumerate(o.ranges):
            f = fleet[g]
            ok = [k for k in range(hi - lo) if o.healthy[lo + k] and o.circuit[lo + k]]
            loads = [int(o.loads[lo + k]) for k in range(hi - lo)]
            assert int(f["n_healthy"]) == len(ok), (tag, g)
            if loads:
                assert (int(f["min_load"]), int(f["max_load"])) == (min(loads), max(loads)), (tag, g)
            if ok:
                k = min(ok, key=lambda k: (loads[k], k))
                assert (int(f["min_load_idx"]), int(f["min_healthy_load"]), int(f["first_healthy"])) == (k, loads[k], ok[0]), (tag, g)
            else:
                assert int(f["min_load_idx"]) == -1 and int(f["first_healthy"]) == -1, (tag, g)


def ragged(reqs):
    offs = np.zeros(len(reqs) + 1, np.uint32)
    np.cumsum([len(r) for r in reqs], out=offs[1:])
    flat = np.concatenate([np.asarray(r, np.uint32) for r in reqs]) if offs[-1] else np.zeros(0, np.uint32)
    return flat.astype(np.uint32), offs


def rand_tokens(rng, n):
    return rng.integers(0, synth.VOCAB, size=n, dtype=np.uint32)


# ---- rank boundaries ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", ["full_tie", "lower_load_first", "bigger_tree_first", "bigger_tree_second"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_rank_boundary_ties(world, variant):
    """Workers b-1 and b sit on both sides of a rank boundary and hold the same sequence: the merge's last-max comparison decides."""
    bs, T = 16, 256
    n = world * 5 + 3                                         # uneven ranges
    f = Fleet(synth.worker_urls(n), world, bs, 8, T)
    try:
        rng = np.random.default_rng(world)
        bounds = [f.oracle.ranges[g][0] for g in range(1, world)]
        loads = np.full(n, 5, np.uint64)
        reqs, expect = [], []
        for b in bounds:
            seq = rand_tokens(rng, T)
            hs = orc.compute_request_content_hashes(seq, bs)
            f.store(b - 1, hs)
            f.store(b, hs)
            if variant == "bigger_tree_first":
                f.store(b - 1, orc.compute_request_content_hashes(rand_tokens(rng, 2 * bs), bs))
            elif variant == "bigger_tree_second":
                f.store(b, orc.compute_request_content_hashes(rand_tokens(rng, 2 * bs), bs))
            elif variant == "lower_load_first":
                loads[b - 1] = 4
            reqs.append(seq)
            expect.append(b - 1 if variant in ("lower_load_first", "bigger_tree_second") else b)
        f.set_state(loads, np.ones(n, np.uint8))
        idx, br = f.check(*ragged(reqs), tag=variant)
        assert list(idx) == expect and set(br.tolist()) == {OVERLAP}
    finally:
        f.close()


# ---- the prologue, re-derived from the summaries ----------------------------------------------------------------------------------------

def _prologue_fleet(world, n, seed=5):
    bs, T = 16, 128
    f = Fleet(synth.worker_urls(n), world, bs, 8, T)
    rng = np.random.default_rng(seed)
    seqs = [rand_tokens(rng, T) for _ in range(12)]
    for s, seq in enumerate(seqs):
        hs = orc.compute_request_content_hashes(seq, bs)
        for g in rng.choice(n, size=min(n, 3), replace=False):
            f.store(int(g), hs[: int(rng.integers(1, len(hs) + 1))])
    reqs = seqs + [rand_tokens(rng, T) for _ in range(6)] + [seqs[0][:40], np.zeros(0, np.uint32)]
    return f, ragged(reqs)


PROLOGUE_STATES = {   # name → (world, n, fn(n, ranges) → loads, healthy, circuit, expected branch set, expected min-load pick or None)
    "equal_min_two_ranks": (4, 22, lambda n, R: ({R[1][0] + 2: 1, R[2][0]: 1}, {}, {}, {OVERLAP, MIN_LOAD}, R[1][0] + 2)),
    "equal_min_first_and_last": (4, 22, lambda n, R: ({R[0][1] - 1: 0, R[3][1] - 1: 0}, {}, {}, {OVERLAP, MIN_LOAD}, R[0][1] - 1)),
    "min_unhealthy": (4, 22, lambda n, R: ({R[0][0]: 0, R[2][0]: 3}, {R[0][0]: 0}, {}, {OVERLAP, MIN_LOAD}, R[2][0])),
    "min_circuit_open": (4, 22, lambda n, R: ({R[1][0]: 0, R[3][0]: 3}, {}, {R[1][0]: 0}, {OVERLAP, MIN_LOAD}, R[3][0])),
    "min_unhealthy_opens_gate": (4, 22, lambda n, R: ({R[0][0]: 0, R[2][0] + 1: 70}, {R[0][0]: 0}, {}, {IMBALANCED}, None)),   # 70 - 10 would not
    "max_circuit_open_opens_gate": (4, 22, lambda n, R: ({R[3][1] - 1: 500}, {}, {R[3][1] - 1: 0}, {IMBALANCED}, None)),
    "max_unhealthy_on_empty_rank_side": (8, 6, lambda n, R: ({5: 300}, {5: 0}, {}, {IMBALANCED}, None)),
    "rank_all_unhealthy": (4, 22, lambda n, R: ({R[1][0]: 1}, {g: 0 for g in range(*R[1])}, {}, {OVERLAP, MIN_LOAD}, None)),
    "empty_ranks": (8, 5, lambda n, R: ({**{g: 70 for g in range(n)}, 3: 60}, {}, {}, {OVERLAP, MIN_LOAD}, 3)),
    "empty_ranks_balanced": (4, 3, lambda n, R: ({g: 100 for g in range(n)}, {}, {}, {OVERLAP, MIN_LOAD}, 0)),
    "empty_and_unhealthy_ranks": (8, 6, lambda n, R: ({g: 90 for g in range(n)}, {0: 0, 1: 0, 2: 0}, {3: 0}, {OVERLAP, MIN_LOAD}, 4)),
    "only_last_rank_healthy": (4, 22, lambda n, R: ({}, {g: 0 for g in range(R[3][0])}, {}, {OVERLAP, MIN_LOAD}, R[3][0])),
    "only_last_rank_healthy_uneven": (4, 6, lambda n, R: ({R[3][0]: 9}, {g: 0 for g in range(R[3][0])}, {}, {OVERLAP, MIN_LOAD}, R[3][0])),
    "no_healthy": (4, 22, lambda n, R: ({}, {g: 0 for g in range(n)}, {}, {NO_HEALTHY}, None)),
    "no_healthy_circuits": (4, 6, lambda n, R: ({}, {}, {g: 0 for g in range(n)}, {NO_HEALTHY}, None)),
}


@pytest.mark.parametrize("name", sorted(PROLOGUE_STATES))
def test_prologue_from_summaries(name):
    world, n, fn = PROLOGUE_STATES[name]
    f, (tokens, offs) = _prologue_fleet(world, n)
    try:
        R = f.oracle.ranges
        load_over, unhealthy, open_circuit, branches, min_pick = fn(n, R)
        loads = np.full(n, 10, np.uint64)
        healthy, circuit = np.ones(n, np.uint8), np.ones(n, np.uint8)
        for g, v in load_over.items():
            loads[g] = v
        for g, v in unhealthy.items():
            healthy[g] = v
        for g, v in open_circuit.items():
            circuit[g] = v
        f.set_state(loads, healthy, circuit)
        idx, br = f.check(tokens, offs, tag=name)
        assert set(br.tolist()) == branches, (name, set(br.tolist()))
        pb, pidx = f.oracle.prologue()
        if min_pick is not None:
            assert pidx == min_pick
            assert int(idx[-1]) == min_pick and int(br[-1]) == MIN_LOAD      # the empty request
        if name == "rank_all_unhealthy":
            assert not any(R[1][0] <= int(i) < R[1][1] for i in idx)
    finally:
        f.close()


def test_f32_gate_across_ranks():
    """The f32 imbalance gate at its rounding edges (tests/test_gpu_pick_thresholds.py's cases), min and max on different ranks of four,
    on healthy, unhealthy and circuit-open workers."""
    from tests import test_gpu_pick_thresholds as M
    W, world = 130, 4
    n_cases = 0
    for abs_thr, rel in M.GATE_CONFIGS:
        cfg = dict(cache_threshold=0.3, balance_abs_threshold=abs_thr, balance_rel_threshold=rel)
        f = Fleet(M.urls_of(W), world, M.PAGE, 64, 1024, cfg=cfg)
        try:
            R = f.oracle.ranges
            layouts = [(R[0][0], R[3][1] - 1, "ok", "ok"), (R[3][1] - 1, R[1][0], "unhealthy", "ok"), (R[2][0], R[0][1] - 1, "ok", "open_circuit"),
                       (R[1][1] - 1, R[2][1] - 1, "open_circuit", "unhealthy")]
            rng = np.random.default_rng(abs_thr)
            for c in (c for c in M.GATE_CASES if (c["abs"], c["rel"]) == (abs_thr, rel)):
                for layout in layouts:
                    loads, healthy, circuit, hot = M.layout_fleet(c, W, layout)
                    req = rand_tokens(rng, 4 * M.PAGE)
                    f.store(hot, orc.compute_request_content_hashes(req, M.PAGE))
                    f.set_state(np.asarray(loads, np.uint64), healthy, circuit)
                    want, imbalanced = M.gate_expectation(c, loads, healthy, circuit, hot)
                    idx, br = f.check(*ragged([req]), tag=(c["name"], layout))
                    assert int(idx[0]) == want and (int(br[0]) == IMBALANCED) == imbalanced, (c["name"], layout)
                    n_cases += 1
        finally:
            f.close()
    assert n_cases == 4 * len(M.GATE_CASES)


# ---- candidate sites ----------------------------------------------------------------------------------------------------------------------

def _site_fleet(per_shard, world, bs, jump, max_blocks, seed):
    """Shards of `per_shard` workers; an index of replicated sequences plus drained requests (the stored prefix is shorter than the jump
    destination) and Multi entries at position 1 (another prefix under the same content)."""
    n = per_shard * world
    T = max_blocks * bs
    f = Fleet(synth.worker_urls(n), world, bs, jump, T)
    rng = np.random.default_rng(seed)
    seqs, blocks = synth_stores("replicas", n, 60, T, bs, seed)
    for g, bl in blocks:
        f.store(g, [h for _, h in bl])
    for s in range(0, 60, 4):                                    # Multi at position 1 for every fourth sequence
        hs = orc.compute_request_content_hashes(seqs[s], bs)
        other = orc.compute_request_content_hashes(rand_tokens(rng, bs), bs)
        f.store(int(rng.integers(0, n)), other + hs[1: int(rng.integers(2, max_blocks + 1))])
    loads = synth.poisson_loads(n, 8, seed)
    healthy = (rng.random(n) > 0.1).astype(np.uint8)
    f.set_state(loads, healthy)
    return f, seqs, rng


def _site_requests(seqs, rng, bs, max_blocks, B, seed):
    tokens, offs = synth_requests(seqs, B, seed, bs, max_blocks * bs)
    reqs = [tokens[offs[i]:offs[i + 1]] for i in range(B)]
    special = [np.zeros(0, np.uint32), seqs[0][: bs - 1], seqs[1][:bs], seqs[2][: min(32, max_blocks) * bs], seqs[3][: max_blocks * bs],
               seqs[4][: min(33, max_blocks) * bs + bs // 2]]
    return ragged(special + reqs)


SITES = [   # (per-shard workers, world, block size, jump, max blocks per request)
    (1, 2, 16, 8, 40), (63, 2, 16, 31, 32), (64, 2, 16, 8, 40), (65, 2, 16, 64, 40), (64, 2, 5, 31, 40), (65, 2, 7, 8, 40),
    (33, 4, 16, 8, 40), (2048, 2, 16, 64, 40), (2048, 2, 3, 8, 24),
]


@pytest.mark.parametrize("per_shard,world,bs,jump,max_blocks", SITES)
def test_candidate_sites(per_shard, world, bs, jump, max_blocks):
    f, seqs, rng = _site_fleet(per_shard, world, bs, jump, max_blocks, seed=per_shard + bs)
    try:
        tokens, offs = _site_requests(seqs, rng, bs, max_blocks, 300, per_shard)
        idx, br = f.check(tokens, offs, tag="mixed")
        assert OVERLAP in br and MIN_LOAD in br
        # the best-overlap worker unhealthy: the winner comes from the next best, possibly on another rank
        loads, healthy = f.oracle.loads.copy(), f.oracle.healthy.copy()
        healthy[idx[br == OVERLAP]] = 0
        f.set_state(loads, healthy)
        f.check(tokens, offs, tag="winners unhealthy")
    finally:
        f.close()


@pytest.mark.parametrize("impl", ["split", "hs", "stream", "fused"])
@pytest.mark.parametrize("per_shard,bs,max_blocks", [(64, 16, 32), (65, 16, 40), (40, 5, 40), (16, 1, 2600)])
def test_candidate_sites_every_path(impl, per_shard, bs, max_blocks):
    """The candidate kernels of each implementation (SMGX_EVENT_PATH): the split pair (search2, or the thread kernel for rows past 160 KB,
    or the warp kernel above 64 workers), the one-launch hash stream, the streaming kernel and the fused kernel."""
    with selected(impl):
        f, seqs, rng = _site_fleet(per_shard, 2, bs, 64 if bs == 1 else 31, max_blocks, seed=7 * per_shard + bs)
        try:
            tokens, offs = _site_requests(seqs, rng, bs, max_blocks, 257, per_shard)
            f.check(tokens, offs, tag=impl)
        finally:
            f.close()


@pytest.mark.parametrize("n", [1, 255, 256, 257, 5000])
def test_batch_sizes(n):
    f, seqs, rng = _site_fleet(65, 4, 16, 8, 40, seed=n)
    try:
        tokens, offs = synth_requests(seqs, n, n, 16, 40 * 16)
        f.check(tokens, offs, tag=n)
    finally:
        f.close()


# ---- the indexes on which the shards depart from the whole fleet --------------------------------------------------------------------------

@pytest.mark.parametrize("impl", ["fused", "split"])
@pytest.mark.parametrize("bs", [4, 16])
@pytest.mark.parametrize("kind", ["count_test", "retain_guard"])
def test_departure_cases(kind, bs, impl):
    case = departure_case(kind, bs)
    with selected(impl):
        f = Fleet([f"http://{nm}:8000" for nm in case["names"]], case["world"], bs, 8, 16 * bs)
        try:
            for g, hs in case["stores"].items():
                f.store(g, hs)
            f.set_state(case["loads"], np.ones(len(case["names"]), np.uint8))
            tokens, offs = ragged([case["tokens"]] * 3)
            idx, br = f.check(tokens, offs, tag=kind)
            widx = f.oracle.select_whole(tokens, offs)[0]
            assert list(idx) == [case["sharded"]] * 3 and list(widx) == [case["whole"]] * 3
        finally:
            f.close()


# ---- requests longer than max_tokens_per_request -------------------------------------------------------------------------------------

@pytest.mark.parametrize("impl", ["fused", "split"])
@pytest.mark.parametrize("world,n_workers", [(2, 40), (4, 3)])
def test_over_length_request(impl, world, n_workers):
    """A request of more than max_blocks blocks: every rank flags it and stores the empty candidate, the merge picks the first min-load
    worker, and each rank's next smgx_synchronize reports SMGX_INVALID_ARGUMENT once — the flag is cleared, the next batch succeeds."""
    from smg_b200 import _lib
    bs, max_blocks = 16, 8
    with selected(impl):
        f = Fleet(synth.worker_urls(n_workers), world, bs, 8, max_blocks * bs)
        try:
            rng = np.random.default_rng(3)
            seqs = [rand_tokens(rng, (max_blocks + 2) * bs) for _ in range(4)]
            for s, seq in enumerate(seqs):
                f.store(s % n_workers, orc.compute_request_content_hashes(seq[: max_blocks * bs], bs))
            loads = np.arange(n_workers, dtype=np.uint64) % 5 + 3
            f.set_state(loads, np.ones(n_workers, np.uint8))
            reqs = [seqs[0][: max_blocks * bs], seqs[1], seqs[2][: max_blocks * bs + bs - 1], seqs[3][: (max_blocks + 1) * bs]]
            tokens, offs = ragged(reqs)
            idx, info, _, _, status = f.run(tokens, offs)
            assert status == [_lib.INVALID_ARGUMENT] * world
            want_i, want_b, want_m = f.oracle.select(tokens, offs, max_blocks)
            assert np.array_equal(idx, want_i) and np.array_equal(info["branch"], want_b) and np.array_equal(info["matched"], want_m)
            pb, pidx = f.oracle.prologue()
            assert list(info["branch"]) == [OVERLAP, MIN_LOAD, OVERLAP, MIN_LOAD] and idx[1] == idx[3] == pidx
            f.check(*ragged(reqs[:1] + reqs[2:3]), tag="after the error")
        finally:
            f.close()
