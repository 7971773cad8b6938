"""Load feedback for prefix_hash and power_of_two (smgx_set_load_feedback_policies with SMGX_FEEDBACK_PREFIX_HASH / _POWER_OF_TWO): a batch is
the request stream of a router that guards every pick (routers/grpc/context.rs:248-259).  Oracle: select_worker one request at a time with the
pick's load bumped after each (tests/feedback_stream.py).  With the bit off, results are bit-equal to frozen batches."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc
from tests import feedback_stream as FS

pytestmark = pytest.mark.gpu


def _workers(urls, loads, healthy=None):
    from smg_b200 import BasicWorker
    ws = [BasicWorker(u) for u in urls]
    for i, w in enumerate(ws):
        w.set_load(int(loads[i]))
        if healthy is not None:
            w.set_healthy(bool(healthy[i]))
    return ws


def _prefix(k=256, factor=1.25, feedback=True):
    from smg_b200 import PrefixHashConfig, PrefixHashPolicy
    pol = PrefixHashPolicy(PrefixHashConfig(prefix_token_count=k, load_factor=factor))
    if feedback:
        pol.set_load_feedback(True)
    return pol, orc.PrefixHashPolicy(k, factor)


def _prefix_check(pol, oph, urls, loads, healthy, ring_urls, reqs, tag):
    ring = pol.hash_ring(ring_urls) if ring_urls is not None else None
    oring = orc.HashRing(ring_urls) if ring_urls is not None else None
    idx, br = pol.select_worker_batch(_workers(urls, loads, healthy), reqs, ring=ring)
    widx, wbr, after = FS.prefix_stream(oph, urls, loads, healthy, oring, reqs)
    assert np.array_equal(idx, widx), (tag, np.nonzero(idx != widx)[0][:5])
    assert br == [orc.PREFIX_BRANCHES[int(b)] for b in wbr], tag
    assert np.array_equal(np.asarray(loads, np.uint64) + np.bincount(idx[idx >= 0], minlength=len(urls)).astype(np.uint64), after), tag
    return idx, np.asarray(br)


def test_prefix_hash_hot_prefix_crosses_the_bound_mid_batch():
    urls = [f"http://worker-{i}.svc:8000" for i in range(64)]
    rng = np.random.default_rng(1)
    pol, oph = _prefix()
    hot = list(rng.integers(0, 128000, size=300))
    reqs = [hot + [i] for i in range(400)] + [list(rng.integers(0, 128000, size=50)) for _ in range(200)]
    reqs = [reqs[i] for i in rng.permutation(len(reqs))]
    idx, br = _prefix_check(pol, oph, urls, rng.integers(0, 20, size=64), [1] * 64, urls, reqs, "hot")
    assert (br == "ring_hit").sum() > 0 and (br == "load_balance_walk").sum() > 100
    frozen, _ = _prefix(feedback=False)
    fidx, fbr = frozen.select_worker_batch(_workers(urls, [5] * 64), [hot + [i] for i in range(100)], ring=frozen.hash_ring(urls))
    assert len(set(fidx)) == 1 and set(fbr) == {"ring_hit"}      # one snapshot: the hot prefix piles onto the ring worker


@pytest.mark.parametrize("factor", [0.8, 0.5, 1.0, 2.0])
def test_prefix_hash_load_factors_unhealthy_and_missing_ring_workers(factor):
    rng = np.random.default_rng(int(factor * 10))
    urls = [f"http://w{i}:8000" for i in range(33)]
    pol, oph = _prefix(k=64, factor=factor)
    ring_urls = urls[:20] + ["http://ghost:1", "http://ghost:2"]
    for rnd in range(3):
        healthy = (rng.random(33) > [0.0, 0.1, 0.5][rnd]).astype(np.uint8)
        reqs = []
        for _ in range(500):
            t = list(rng.integers(0, 128000, size=int(rng.integers(0, 200))))
            prev = [r for r in reqs if r is not None]
            if prev and rng.random() < 0.5:
                t = prev[int(rng.integers(0, len(prev)))][:64] + t
            reqs.append(t if rng.random() > 0.02 else None)
        _prefix_check(pol, oph, urls, rng.integers(0, [1, 10, 300][rnd], size=33), healthy, ring_urls, reqs, (factor, rnd))


def test_prefix_hash_without_ring_is_a_least_loaded_stream():
    urls = [f"http://w{i}:8000" for i in range(8)]
    pol, oph = _prefix()
    idx, br = _prefix_check(pol, oph, urls, [0] * 8, [1] * 8, None, [[i, i + 1] for i in range(16)], "no ring")
    assert list(idx) == list(range(8)) * 2 and set(br) == {"fallback_least_load"}


def test_prefix_hash_running_total_above_2_pow_53():
    urls = [f"http://w{i}:8000" for i in range(5)]
    rng = np.random.default_rng(3)
    pol, oph = _prefix()
    loads = (np.uint64(1) << np.uint64(53)) + rng.integers(0, 4096, size=5).astype(np.uint64)
    hot = list(range(1, 40))
    reqs = [hot] * 300 + [list(rng.integers(0, 9999, size=20)) for _ in range(300)]
    _prefix_check(pol, oph, urls, loads, [1] * 5, urls, reqs, "2^53")


def test_prefix_hash_three_device_batches_form_one_stream():
    from smg_b200 import _lib
    rng = np.random.default_rng(9)
    urls = [f"http://w{i}:8000" for i in range(64)]
    pol, oph = _prefix()
    ring, oring = pol.hash_ring(urls), orc.HashRing(urls)
    loads = rng.integers(0, 30, size=64)
    ws = _workers(urls, loads)
    h, model = pol._h, pol._push_fleet(ws, ring)
    hot = list(rng.integers(0, 128000, size=256))
    batches = []
    for b in range(3):
        reqs = [(hot if rng.random() < 0.5 else []) + list(rng.integers(0, 128000, size=int(rng.choice([61, 255, 301])))) for _ in range(300)]
        batches.append(reqs)
    err = _lib.new_err()
    L = h.L
    d_tok, d_off, d_out = [], [], []
    for reqs in batches:
        tokens = np.concatenate([np.asarray(r, np.uint32) for r in reqs])
        off = np.zeros(len(reqs) + 1, np.uint32)
        np.cumsum([len(r) for r in reqs], out=off[1:])
        for arr, lst in ((tokens, d_tok), (off, d_off)):
            ptr = L.smgx_device_alloc(h.p, arr.nbytes, C.byref(err))
            h.call("smgx_memcpy_h2d", ptr, arr.ctypes.data_as(C.c_void_p), arr.nbytes)
            lst.append(ptr)
        d_out.append(L.smgx_device_alloc(h.p, len(reqs) * 4, C.byref(err)))
    vp = C.c_void_p * 3
    h.call("smgx_prefix_hash_select_many_tokens_device", model, 3, vp(*d_tok), vp(*d_off), (C.c_uint32 * 3)(*[len(r) for r in batches]), vp(*d_out))
    h.call("smgx_synchronize")
    want, wbr, _ = FS.prefix_stream(oph, urls, loads, [1] * 64, oring, [r for reqs in batches for r in reqs])
    assert (wbr == orc.PREFIX_BRANCHES.index("load_balance_walk")).sum() > 0
    for k in range(3):
        got = np.zeros(300, np.int32)
        h.call("smgx_memcpy_d2h", got.ctypes.data_as(C.c_void_p), d_out[k], got.nbytes)
        assert np.array_equal(got, want[300 * k: 300 * (k + 1)]), k
    for ptr in d_tok + d_off + d_out:
        L.smgx_device_free(h.p, ptr)


@pytest.mark.parametrize("n_workers", [1, 2, 3, 64, 257, 4096])
def test_power_of_two_stream_matches_one_by_one_oracle(n_workers):
    from smg_b200 import PowerOfTwoPolicy
    rng = np.random.default_rng(n_workers)
    urls = [f"http://w{i}:8000" for i in range(n_workers)]
    pol, op2 = PowerOfTwoPolicy(), orc.PowerOfTwoPolicy()
    pol.set_load_feedback(True)
    cached = {u: float(rng.random()) for u in urls if rng.random() < 0.5}      # mixed: some pairs compare token usage, most request counts
    pol.update_loads(cached); op2.update_loads(cached)
    n = 1500 if n_workers > 64 else 3000
    for rnd in range(2):
        loads = rng.integers(0, [8, 1 << 60][rnd], size=n_workers).astype(np.uint64)
        healthy = (rng.random(n_workers) > 0.1).astype(np.uint8) if n_workers > 3 else np.ones(n_workers, np.uint8)
        seed = int(rng.integers(0, 2**63))
        idx, pairs, metric = pol.select_worker_batch(_workers(urls, loads, healthy), n, seed=seed, with_details=True)
        widx, wpairs, wmetric, after = FS.p2c_stream(op2, urls, loads, healthy, [1] * n_workers, n, seed)
        assert np.array_equal(idx, widx) and np.array_equal(pairs, wpairs) and np.array_equal(metric, wmetric), (rnd, np.nonzero(idx != widx)[0][:5])
        assert np.array_equal(loads + np.bincount(idx[idx >= 0], minlength=n_workers).astype(np.uint64), after)


def test_feedback_off_is_bit_equal_for_prefix_hash_and_power_of_two():
    from smg_b200 import PowerOfTwoPolicy
    rng = np.random.default_rng(4)
    urls = [f"http://w{i}:8000" for i in range(40)]
    loads = rng.integers(0, 50, size=40)
    reqs = [list(rng.integers(0, 500, size=int(rng.integers(1, 40)))) for _ in range(800)]
    out = []
    for how in ("never", "mask0", "event_only"):
        pol, _ = _prefix(feedback=False)
        p2 = PowerOfTwoPolicy()
        for p, bit in ((pol, 2), (p2, 4)):
            if how == "mask0":
                p._h.call("smgx_set_load_feedback_policies", bit)
                p._h.call("smgx_set_load_feedback_policies", 0)
            if how == "event_only":
                p._h.call("smgx_set_load_feedback_policies", 7)
                p._h.call("smgx_set_load_feedback", 1)
        idx, br = pol.select_worker_batch(_workers(urls, loads), reqs, ring=pol.hash_ring(urls))
        pidx, ppairs, pmetric = p2.select_worker_batch(_workers(urls, loads), 800, seed=99, with_details=True)
        out.append((idx.tolist(), br, pidx.tolist(), ppairs.tolist(), pmetric.tolist()))
    assert out[0] == out[1] == out[2]
