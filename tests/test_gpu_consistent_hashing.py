"""consistent_hashing on the GPU (smgx_consistent_hashing_select_batch) against the oracle (tests/consistent_hashing_oracle.py): picks,
branches and key positions bit for bit on seeded batches, the reference's unit tests through PolicyFactory, and the golden key positions
of the independent `blake3` package, multi-chunk keys included."""
import importlib.util
import json
import os

import numpy as np
import pytest

from tests import consistent_hashing_oracle as ch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("gen_ch_golden", os.path.join(HERE, "golden", "gen_consistent_hashing_golden.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "consistent_hashing_vectors.json")))


def _workers(urls, healthy=None, circuit=None):
    from smg_b200 import BasicWorker
    ws = [BasicWorker(u) for u in urls]
    for i, w in enumerate(ws):
        if healthy is not None:
            w.set_healthy(bool(healthy[i]))
        if circuit is not None:
            w.set_circuit_ok(bool(circuit[i]))
    return ws


def _policy(**kw):
    from smg_b200 import PolicyFactory
    return PolicyFactory.create_by_name("consistent_hashing", **kw)


def _info(ring=None, **headers):
    from smg_b200 import SelectWorkerInfo
    return SelectWorkerInfo(headers=headers or None, hash_ring=ring)


# ---- the reference's unit tests (consistent_hashing.rs:198-532) through the product ----
def test_reference_unit_tests_through_the_product():
    pol = _policy()
    assert pol.name() == "consistent_hashing"
    w3 = _workers(["http://w1:8000", "http://w2:8000", "http://w3:8000"])
    w2 = _workers(["http://w1:8000", "http://w2:8000"])
    # test_consistent_routing
    first, _ = pol.select_worker_impl(w3, _info(**{"x-smg-routing-key": "user-123"}))
    for _ in range(10):
        assert pol.select_worker_impl(w3, _info(**{"x-smg-routing-key": "user-123"})) == (first, "routing_key_hit")
    # test_different_keys_distribute
    assert len({pol.select_worker(w3, _info(**{"x-smg-routing-key": f"user-{i}"})) for i in range(100)}) > 1
    # test_target_worker_hit / miss out of bounds / priority over routing key
    assert pol.select_worker_impl(w2, _info(**{"x-smg-target-worker": "1"})) == (1, "target_worker_hit")
    assert pol.select_worker_impl(w2, _info(**{"x-smg-target-worker": "5"})) == (None, "target_worker_miss")
    assert pol.select_worker_impl(w2, _info(**{"x-smg-target-worker": "1", "x-smg-routing-key": "some-key"})) == (1, "target_worker_hit")
    # test_target_worker_miss_unhealthy
    assert pol.select_worker_impl(_workers(["http://w1:8000", "http://w2:8000"], [1, 0]), _info(**{"x-smg-target-worker": "1"})) == (None, "target_worker_miss")
    # test_fallback_random_distribution
    dist = set()
    for _ in range(100):
        idx, br = pol.select_worker_impl(w3, _info())
        assert idx is not None and br == "random_fallback"
        dist.add(idx)
    assert len(dist) > 1
    # test_no_healthy_workers / test_empty_workers
    assert pol.select_worker_impl(_workers(["http://w1:8000"], [0]), _info(**{"x-smg-routing-key": "test"})) == (None, "no_healthy_workers")
    assert pol.select_worker_impl([], _info()) == (None, "no_healthy_workers")
    # test_consistent_hash_minimal_redistribution
    urls4 = [f"http://w{i}:8000" for i in range(4)]
    w4 = _workers(urls4)
    ring = pol.hash_ring(urls4)
    before = {i: pol.select_worker(w4, _info(ring, **{"x-smg-routing-key": f"user-{i}"})) for i in range(100)}
    w4[1].set_healthy(False)
    moved = sum(pol.select_worker(w4, _info(ring, **{"x-smg-routing-key": f"user-{i}"})) != before[i] for i in range(100))
    assert moved <= sum(v == 1 for v in before.values()) + 5 and moved < 50
    # test_routing_key_failover_and_recovery
    urls3 = [f"http://w{i}:8000" for i in range(3)]
    ws = _workers(urls3)
    ring3 = pol.hash_ring(urls3)
    info = _info(ring3, **{"x-smg-routing-key": "session-abc-123"})
    orig = pol.select_worker(ws, info)
    ws[orig].set_healthy(False)
    fail = pol.select_worker(ws, info)
    assert fail != orig and ws[fail].is_healthy()
    assert all(pol.select_worker(ws, info) == fail for _ in range(5))
    ws[orig].set_healthy(True)
    assert pol.select_worker(ws, info) == orig
    # test_empty_routing_key_uses_fallback
    idx, br = pol.select_worker_impl(w2, _info(**{"x-smg-routing-key": ""}))
    assert idx is not None and br == "random_fallback"


# ---- golden key positions through out_key_pos ----
def test_golden_key_positions():
    pol = _policy()
    urls = [f"http://worker-{i}:8000" for i in range(5)]
    ws = _workers(urls)
    keys = [k for k in GOLDEN["keys"] if k["len"] > 0]
    hs = [{"x-smg-routing-key": gen.key_bytes(k["len"], k["salt"])} for k in keys]
    hs += [{"cookie": gen.key_bytes(k["len"], k["salt"])} for k in keys]
    for ring in (None, pol.hash_ring(urls)):
        idx, br, kp = pol.select_worker_batch(ws, hs, ring=ring, seed=1, with_details=True)
        want = [int(k["pos"]) for k in keys] * 2
        assert [int(x) for x in kp] == want
        assert set(br) == {"routing_key_hit"}


def test_golden_no_ring_decisions():
    pol = _policy()
    for d in GOLDEN["no_ring_decisions"]:
        ws = _workers(d["urls"], d["healthy"])
        hs = [{"x-smg-routing-key": gen.key_bytes(r["len"], r["salt"])} for r in d["requests"]]
        idx, br, kp = pol.select_worker_batch(ws, hs, seed=0, with_details=True)
        assert idx.tolist() == [r["idx"] for r in d["requests"]]
        assert [int(x) for x in kp] == [int(r["pos"]) for r in d["requests"]]


# ---- seeded batches against the oracle ----
def _value(rng, h, w):
    """A header value for header h: valid, empty, obs-text or control bytes."""
    u = rng.random()
    if u < 0.08:
        return b""
    if u < 0.14:
        return "é".encode() + b"x"
    if u < 0.17:
        return b"a\x01b"
    if h == 0:
        return rng.choice([str(int(rng.integers(0, w + 2))).encode(), b"+" + str(int(rng.integers(0, w))).encode(), b"00" + str(int(rng.integers(0, w))).encode(),
                           b"-0", b"+", b" 1", b"18446744073709551615", b"18446744073709551616", b"x"])
    if h == 4 and rng.random() < 0.3:
        n = int(rng.integers(1, 41)) * 1024 - int(rng.integers(0, 1024))   # 1 to 40 chunks
    else:
        n = int(rng.choice([1, 5, 36, 63, 64, 65, 200, 1023, 1024]))
    return gen.key_bytes(n, int(rng.integers(0, 1 << 30)))


def _batch(rng, n, w, mix):
    hs = []
    for _ in range(n):
        if rng.random() < 0.05:
            hs.append(None)
            continue
        row = [None] * 5
        for h in range(5):
            if rng.random() < mix[h]:
                row[h] = _value(rng, h, w)
        hs.append(row)
    return hs


def _pack(hs, pad):
    blob, offs, present = bytearray(b"\x00" * pad), [pad], []
    for row in hs:
        bits = 0
        for h in range(5):
            v = None if row is None else row[h]
            if v is not None:
                bits |= 1 << h
                blob += v
            offs.append(len(blob))
        present.append(bits)
    return bytes(blob) + b"\xff" * 3, offs, present


def _fleet(rng, w):
    urls = [f"http://worker-{i}:8000" for i in range(w)]
    for i in range(w):
        if w > 1 and rng.random() < 0.1:
            urls[i] = urls[int(rng.integers(0, w))]                    # duplicate URLs
    healthy = (rng.random(w) > 0.25).astype(np.uint8)
    circuit = (rng.random(w) > 0.3).astype(np.uint8)                  # not read by this policy
    return urls, healthy, circuit


@pytest.mark.parametrize("w,n,seed", [(1, 500, 1), (2, 2000, 2), (3, 3000, 3), (17, 5000, 4), (64, 8000, 5), (512, 4000, 6), (4096, 3000, 7)])
def test_random_fleets_equal_oracle(w, n, seed):
    rng = np.random.default_rng(seed)
    pol = _policy()
    mixes = [(0.1, 0.5, 0.3, 0.2, 0.3), (0.0, 0.0, 0.0, 0.0, 0.0), (0.3, 0.3, 0.3, 0.3, 0.3)]
    for rnd, ring_kind in enumerate(("ring", "none", "empty", "partial", "ring")):
        urls, healthy, circuit = _fleet(rng, w)
        ws = _workers(urls, healthy, circuit)
        uniq = list(dict.fromkeys(urls))
        ring_urls = {"ring": uniq, "none": None, "empty": [], "partial": uniq[: max(1, len(uniq) // 2)] + ["http://elsewhere:1"]}[ring_kind]
        ring = None if ring_urls is None else pol.hash_ring(ring_urls)
        oring = None if ring_urls is None else ch.Ring(ring_urls)
        hs = _batch(rng, n, w, mixes[rnd % 3])
        pad = int(rng.integers(0, 50))
        values, offs, present = _pack(hs, pad)
        s = int(rng.integers(0, 2**63))
        idx, br, kp = pol.select_worker_batch(ws, ring=ring, seed=s, with_details=True, values=values, offsets=offs, present=present)
        oidx, obr, okp = ch.select_batch(urls, healthy.tolist(), oring, hs, s)
        assert idx.tolist() == oidx, ring_kind
        assert br == obr, ring_kind
        assert kp.astype(np.uint64).tolist() == okp, ring_kind
        cidx, cbr, ckp, _ = ch.cpp_select_batch(urls, healthy.tolist(), ring_urls, values, offs, present, s, threads=4)
        assert np.array_equal(idx, cidx) and br == cbr and np.array_equal(kp, ckp), ring_kind


def test_large_batch_and_offsets_not_from_zero():
    rng = np.random.default_rng(11)
    pol = _policy(max_batch=70000)
    urls, healthy, circuit = _fleet(rng, 64)
    ws = _workers(urls, healthy, circuit)
    ring = pol.hash_ring(list(dict.fromkeys(urls)))
    oring = ch.Ring(list(dict.fromkeys(urls)))
    n = 70_001
    hs = _batch(rng, n, 64, (0.05, 0.6, 0.2, 0.1, 0.2))
    values, offs, present = _pack(hs, 1000)
    idx, br, kp = pol.select_worker_batch(ws, ring=ring, seed=3, with_details=True, values=values, offsets=offs, present=present)
    oidx, obr, okp = ch.select_batch(urls, healthy.tolist(), oring, hs, 3)
    assert idx.tolist() == oidx and br == obr and kp.astype(np.uint64).tolist() == okp
    assert {"target_worker_hit", "target_worker_miss", "routing_key_hit", "random_fallback"} <= set(obr)


def test_pick_only_matches_details():
    rng = np.random.default_rng(5)
    pol = _policy()
    urls, healthy, _ = _fleet(rng, 17)
    ws = _workers(urls, healthy)
    hs = _batch(rng, 3000, 17, (0.1, 0.5, 0.3, 0.2, 0.3))
    packed = dict(zip(("values", "offsets", "present"), _pack(hs, 0)))
    a = pol.select_worker_batch(ws, seed=9, **packed)
    b, _, _ = pol.select_worker_batch(ws, seed=9, with_details=True, **packed)
    c = pol.select_worker_batch(ws, [None if r is None else {ch.HEADERS[h]: v for h, v in enumerate(r) if v is not None} for r in hs], seed=9)
    assert np.array_equal(a, b) and np.array_equal(a, c)


def test_invalid_arguments():
    from smg_b200 import SmgxError
    pol = _policy()
    ws = _workers(["http://a", "http://b"])
    with pytest.raises(SmgxError):
        pol.select_worker_batch(ws, values=b"abc", offsets=[0, 1, 2, 3, 2, 3], present=[31])   # decreasing offsets
    big = b"k" * ((2 << 20) + 1)
    with pytest.raises(SmgxError):
        pol.select_worker_batch(ws, [{"cookie": big}])
    assert pol.select_worker_batch(ws, [{"x-smg-target-worker": big}]).tolist() == [-1]   # the target worker is parsed, not hashed


@pytest.mark.parametrize("pad", [0, 1, 2, 3])
def test_rejected_byte_in_word_scan(pad):
    """HeaderValue::to_str on values long enough for the word-at-a-time scan: a rejected byte at every residue mod 4 and at aligned middle
    offsets, in targets (→ the routing key decides) and in implicit keys up to 1500 bytes (→ the random fallback)."""
    pol = _policy()
    urls = [f"http://worker-{i}:8000" for i in range(5)]
    ws = _workers(urls)
    hs = []
    for n in (9, 64, 1500):
        base = b"k" * n
        for at in sorted({0, 1, 2, 3, 4, 5, 6, 7, n // 2 - n // 2 % 4, n // 2 - n // 2 % 4 + 1, n - 4, n - 3, n - 2, n - 1}):
            for bad in (0x80, 0x01):
                v = base[:at] + bytes([bad]) + base[at + 1:]
                hs += [[v, b"abc", None, None, None], [None, None, None, None, v], [None, v, base, None, None], [None, None, v, base, None]]
    values, offs, present = _pack(hs, pad)
    idx, br, kp = pol.select_worker_batch(ws, seed=17, with_details=True, values=values, offsets=offs, present=present)
    oidx, obr, okp = ch.select_batch(urls, [1] * 5, None, hs, 17)
    assert idx.tolist() == oidx and br == obr and kp.astype(np.uint64).tolist() == okp
    assert obr[0::4] == ["routing_key_hit"] * (len(hs) // 4) and obr[1::4] == ["random_fallback"] * (len(hs) // 4)
    assert obr[2::4] == ["routing_key_hit"] * (len(hs) // 4) and obr[3::4] == ["random_fallback"] * (len(hs) // 4)
