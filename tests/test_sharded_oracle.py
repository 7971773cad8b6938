"""The per-shard oracle of the worker-id-sharded pick (tests/sharded_oracle.py) against the whole-fleet oracle, on the CPU.

The sharded pick runs the reference jump search on each shard's index alone; on crafted indexes this departs from the whole-fleet
search (the count test and the retain guard compare sizes of whole-fleet worker sets).  On indexes where every (position, content)
entry holds workers of one prefix chain, nested by depth — how the sharded tests and bench.py's config-4 leg build them — the two
agree, which is what keeps bench.py's whole-fleet parity check of the sharded leg valid."""
import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth
from tests.sharded_oracle import (IMBALANCED, MIN_LOAD, NO_HEALTHY, OVERLAP, ShardedOracle, departure_case, seq_blocks, synth_requests,
                                  synth_stores)

CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5)


def _oracle_for(case, bs):
    urls = [f"http://{nm}:8000" for nm in case["names"]]
    o = ShardedOracle(urls, case["world"], 8, dict(CFG, block_size=bs))
    sid = 1
    for g, hs in case["stores"].items():
        o.apply_stored(g, seq_blocks(hs, sid))
        sid += 100
    o.set_state(case["loads"], np.ones(len(urls), np.uint8))
    return o


@pytest.mark.parametrize("bs", [4, 16])
@pytest.mark.parametrize("kind", ["count_test", "retain_guard"])
def test_departure_from_whole_fleet(kind, bs):
    case = departure_case(kind, bs)
    o = _oracle_for(case, bs)
    off = np.array([0, case["tokens"].size])
    idx, br, ma = o.select(case["tokens"], off)
    widx, wbr, wma = o.select_whole(case["tokens"], off)
    assert (int(idx[0]), int(br[0])) == (case["sharded"], OVERLAP)
    assert (int(widx[0]), int(wbr[0])) == (case["whole"], OVERLAP)
    assert idx[0] != widx[0]
    hashes = orc.compute_request_content_hashes(case["tokens"], bs)
    a, d = case["names"].index("A"), case["names"].index("D")
    whole_scores = o.whole.find_matches(hashes)[0]
    per_shard = {g: o.candidate(o.rank_of(g), hashes) for g in (a, d)}
    if kind == "count_test":
        assert whole_scores[a] == whole_scores[d] == 9        # the count test at position 8 passes on sizes alone
        assert per_shard[a][0] == 9 and per_shard[d][0] == 8  # D's shard has no entry at position 8
        assert int(ma[0]) == int(wma[0]) == 9
    else:
        assert whole_scores[a] == whole_scores[d] == 5        # position 4's Single set {X1, X2} is not smaller than {A, D}
        assert per_shard[a][0] == 4 and per_shard[d][0] == 5  # A's shard holds no X: A is dropped at position 4
        assert int(ma[0]) == int(wma[0]) == 5


def test_departure_needs_the_split():
    """The same index in ONE shard is the whole-fleet search: the departure comes from the split alone."""
    for kind in ("count_test", "retain_guard"):
        case = departure_case(kind, 4)
        urls = [f"http://{nm}:8000" for nm in case["names"]]
        o = ShardedOracle(urls, 1, 8, dict(CFG, block_size=4))
        sid = 1
        for g, hs in case["stores"].items():
            o.apply_stored(g, seq_blocks(hs, sid))
            sid += 100
        o.set_state(case["loads"], np.ones(len(urls), np.uint8))
        off = np.array([0, case["tokens"].size])
        assert int(o.select(case["tokens"], off)[0][0]) == int(o.select_whole(case["tokens"], off)[0][0]) == case["whole"]


def _fleet_round(n, seed, kind):
    rng = np.random.default_rng(seed + 99)
    loads = synth.poisson_loads(n, 8, seed)
    healthy = (rng.random(n) > 0.15).astype(np.uint8)
    circuit = (rng.random(n) > 0.05).astype(np.uint8)
    if kind == "imbalanced":
        loads[n // 2] += 500
    elif kind == "none":
        healthy[:] = 0
    return loads, healthy, circuit


@pytest.mark.parametrize("stores", ["replicas", "config4"])
@pytest.mark.parametrize("world,n_workers", [(2, 48), (4, 130), (8, 259)])
def test_synth_indexes_match_whole_fleet(stores, world, n_workers):
    bs, T, jump, B = 16, 256, 8, 240
    seed = world * 1000 + n_workers
    seqs, blocks = synth_stores(stores, n_workers, 120, T, bs, seed)
    o = ShardedOracle(synth.worker_urls(n_workers), world, jump, dict(CFG, block_size=bs))
    for g, bl in blocks:
        o.apply_stored(g, bl)
    seen = set()
    for r, kind in enumerate(["balanced", "balanced", "imbalanced", "none"]):
        o.set_state(*_fleet_round(n_workers, seed + r, kind))
        tokens, offs = synth_requests(seqs, B, seed + r, bs, T)
        idx, br, ma = o.select(tokens, offs)
        widx, wbr, wma = o.select_whole(tokens, offs)
        assert np.array_equal(idx, widx) and np.array_equal(br, wbr)
        ev = br == OVERLAP
        assert np.array_equal(ma[ev], wma[ev])
        seen |= set(br.tolist())
    assert {OVERLAP, MIN_LOAD, IMBALANCED, NO_HEALTHY} <= seen
