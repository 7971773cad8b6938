"""CPU checks of the tree-mode request stream with load feedback: the oracle stream on hand cases, and the switch's argument checks on a
host-mirror policy (device_id = -1)."""
import numpy as np
import pytest

from oracle import orc
from smg_b200 import _lib
from tests import feedback_stream as FS

CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=16)


def _oracle(n):
    orc.reset_globals()
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **CFG)
    urls = [f"http://w{i}:8000" for i in range(n)]
    op.set_workers(urls)
    return op, urls


def test_equal_loads_novel_texts_go_round_robin():
    op, _ = _oracle(4)
    texts = [f"{c} is a request no other request starts with" for c in "ABCDEFGH"]
    idx, br, _, _, after = FS.stream(op, [0] * 4, texts=texts)
    assert list(idx) == [0, 1, 2, 3, 0, 1, 2, 3]
    assert set(br) == {FS.BR["tree_min_load"]}
    assert list(after) == [2, 2, 2, 2]
    frozen, _, _, _ = op.select_batch_text([f"{c} again, one snapshot" for c in "IJKLMNOP"])[:4]
    assert set(frozen) == {0}          # without the bumps every min-load request lands on the first least loaded worker


def test_equal_loads_novel_token_requests_go_round_robin():
    op, _ = _oracle(4)
    reqs = [[1000 + 37 * i + k for k in range(40)] for i in range(8)]
    idx, br, _, _, after = FS.stream(op, [0] * 4, requests=reqs)
    assert list(idx) == [0, 1, 2, 3, 0, 1, 2, 3]
    flat = np.concatenate([np.asarray(r, np.uint32) for r in reqs])
    offs = np.arange(9, dtype=np.uint64) * 40
    op2, _ = _oracle(4)
    idx2, br2, _, loads2 = op2.select_batch_tokens_feedback(flat, offs)   # the token stream the event tests use agrees
    assert list(idx2) == list(idx) and list(br2) == list(br) and list(loads2) == list(after)


def test_gate_closes_after_the_computed_number_of_picks():
    """Three workers at 0, one at 100 (abs 64, rel 1.5): the gate stays open while 100 - min > 64, i.e. until the three least loaded
    workers reach 36 each — 108 water-filling picks — and is closed for request 108."""
    op, _ = _oracle(4)
    loads = [0, 0, 0, 100]
    closes_at = 3 * next(m for m in range(200) if not (100 - m > 64 and float(np.float32(100)) > float(np.float32(m) * np.float32(1.5))))
    assert closes_at == 108
    texts = [f"request {i:04d} with its own text" for i in range(130)]
    idx, br, _, _, after = FS.stream(op, loads, texts=texts)
    assert set(br[:closes_at]) == {FS.BR["imbalanced_min_load"]}
    assert FS.BR["imbalanced_min_load"] not in set(br[closes_at:])
    assert list(idx[:6]) == [0, 1, 2, 0, 1, 2]
    assert list(after[:3]) == [36 + int((idx[closes_at:] == w).sum()) for w in range(3)] and after[3] == 100 + (idx == 3).sum()


def test_unhealthy_worker_pins_the_minimum_and_keeps_the_gate_open():
    op, _ = _oracle(4)
    op.set_state(healthy=[1, 1, 1, 0])
    idx, br, _, _, after = FS.stream(op, [10, 10, 10, 0], texts=[f"{i} text" for i in range(300)])
    # min over ALL workers stays 0 (the unhealthy worker is never picked): once a healthy worker reaches 65 the gate opens for good
    first = int(np.argmax(br == FS.BR["imbalanced_min_load"]))
    assert first >= 150 and set(br[first:]) == {FS.BR["imbalanced_min_load"]}
    assert 3 not in set(idx) and after[3] == 0


def test_tenant_outside_the_slice_bumps_first_healthy_without_insert():
    op, _ = _oracle(3)
    op.string_tree().insert_text("shared system prompt, long enough to match", "http://gone:1")
    before = op.string_tree().entries()
    idx, br, _, _, after = FS.stream(op, [5, 0, 0], texts=["shared system prompt, long enough to match"] * 3)
    assert list(br) == [FS.BR["tree_fallback_first_healthy"]] * 3 and list(idx) == [0, 0, 0]
    assert list(after) == [8, 0, 0]
    assert [k for k, _ in op.string_tree().entries()] == [k for k, _ in before]


def _host_policy(mode="sequential"):
    from smg_b200 import CacheAwareConfig, CacheAwarePolicy
    return CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0), device_id=-1, tree_batch_mode=mode)


def test_mask_validation_on_a_host_mirror_policy():
    pol = _host_policy()
    for mask in (0, 1, 2, 4, 7, 6, 0):
        pol._h.call("smgx_set_load_feedback_policies", mask)
    for bad in (8, 9, 0x80000000, 0xFFFFFFFF):
        with pytest.raises(_lib.SmgxError) as e:
            pol._h.call("smgx_set_load_feedback_policies", bad)
        assert e.value.code == _lib.INVALID_ARGUMENT
    pol.set_load_feedback_all_modes(True)
    pol.set_load_feedback(True)
    pol.set_load_feedback(False)


def test_snapshot_tree_batches_refuse_cache_aware_feedback():
    pol = _host_policy("snapshot")
    with pytest.raises(_lib.SmgxError) as e:
        pol.set_load_feedback_all_modes(True)
    assert e.value.code == _lib.INVALID_ARGUMENT and "SNAPSHOT" in e.value.msg
    pol._h.call("smgx_set_load_feedback_policies", 6)   # prefix_hash and power_of_two have no tree: fine in either tree batch mode
    pol.set_load_feedback(True)              # the event-driven switch keeps its meaning in either tree batch mode
    pol.set_load_feedback_all_modes(False)
    seq = _host_policy()
    seq.set_load_feedback_all_modes(True)
    seq.set_tree_batch_mode("snapshot")      # accepted here; a tree-mode call that meets the combination refuses it


def test_prefix_hash_ring_worker_crosses_the_bound():
    """5 workers at load 4 (Σ 20, load_factor 1.25): after k picks of the ring worker the bound is (21 + k) / 5 × 1.25 = (21 + k) / 4 and its
    load 4 + k, so it passes load_ok for k = 0, 1 (3k ≤ 5) and the walk sends request 2 to the least loaded worker."""
    oph = orc.PrefixHashPolicy(256, 1.25)
    urls = [f"http://w{i}:8000" for i in range(5)]
    ring = orc.HashRing(urls)
    hot = [11, 22, 33, 44]
    idx, br, after = FS.prefix_stream(oph, urls, [4] * 5, [1] * 5, ring, [hot] * 8)
    ringw = idx[0]
    assert list(br[:2]) == [orc.PREFIX_BRANCHES.index("ring_hit")] * 2 and set(idx[:2]) == {ringw}
    assert br[2] == orc.PREFIX_BRANCHES.index("load_balance_walk") and idx[2] != ringw
    assert int(after.sum()) == 20 + 8
    frozen, fbr, _ = oph.select_batch(urls, [4] * 5, [1] * 5, ring, np.array(hot * 8, np.uint32), np.arange(9, dtype=np.uint64) * 4)
    assert set(frozen) == {ringw}      # one snapshot: every request of the hot prefix lands on the ring worker


def test_power_of_two_stream_compares_running_loads():
    op2 = orc.PowerOfTwoPolicy()
    urls = [f"http://w{i}:8000" for i in range(2)]
    idx, pairs, metric, after = FS.p2c_stream(op2, urls, [0, 0], [1, 1], [1, 1], 10, 77)
    assert set(metric) == {0} and list(after) == [5, 5]    # two workers: every request compares both, the running loads alternate them
    fidx, fpairs, _, _ = op2.select_batch(urls, [0, 0], [1, 1], [1, 1], 10, 77)
    assert np.array_equal(fpairs, pairs)                  # same draws
