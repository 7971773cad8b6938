"""CPU: the consistent_hashing oracles — the C++ restatement (tests/cpp/consistent_hashing_oracle.h) and the Python one
(tests/consistent_hashing_oracle.py) — against the reference's own unit tests (consistent_hashing.rs:198-532, hash_ring.rs tests), one
explicit case per rule, the golden vectors written by tests/golden/gen_consistent_hashing_golden.py with the independent `blake3`
package, and each other on seeded batches."""
import importlib.util
import json
import os

import pytest

from tests import consistent_hashing_oracle as ch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "consistent_hashing_vectors.json")
_spec = importlib.util.spec_from_file_location("gen_ch_golden", os.path.join(HERE, "golden", "gen_consistent_hashing_golden.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)


def hdr(target=None, key=None, auth=None, xff=None, cookie=None):
    enc = lambda v: v.encode() if isinstance(v, str) else v   # noqa: E731
    return [enc(target), enc(key), enc(auth), enc(xff), enc(cookie)]


IMPL = "python"


@pytest.fixture(autouse=True, params=["python", "cpp"])
def impl(request):
    """Every decision test runs on the Python restatement and on the C++ one (tests/cpp/consistent_hashing_oracle.h)."""
    global IMPL
    IMPL = request.param
    yield request.param
    IMPL = "python"


def decide(urls, healthy, headers, ring=None, seed=7, i=0):
    if IMPL == "python":
        return ch.select_worker(urls, healthy, ring, headers, seed, i)
    # request i of a batch draws draw i: the request goes last in a batch of i + 1
    values, offs, present = ch.pack([None] * i + [headers])
    idx, br, kp, _ = ch.cpp_select_batch(urls, healthy, None if ring is None else ring.urls, values, offs, present, seed)
    return (None if idx[-1] < 0 else int(idx[-1])), br[-1], int(kp[-1])


def pick(urls, healthy, headers, ring=None, seed=7, i=0):
    idx, br, _ = decide(urls, healthy, headers, ring, seed, i)
    return idx, br


W3 = ["http://w1:8000", "http://w2:8000", "http://w3:8000"]
W2 = ["http://w1:8000", "http://w2:8000"]


# ---- consistent_hashing.rs tests ----
def test_consistent_routing():
    first, _ = pick(W3, [1, 1, 1], hdr(key="user-123"))
    for _ in range(10):
        assert pick(W3, [1, 1, 1], hdr(key="user-123")) == (first, "routing_key_hit")


def test_different_keys_distribute():
    dist = {pick(W3, [1, 1, 1], hdr(key=f"user-{i}"))[0] for i in range(100)}
    assert len(dist) > 1


def test_target_worker_hit():
    assert pick(W2, [1, 1], hdr(target="1")) == (1, "target_worker_hit")


def test_target_worker_miss_out_of_bounds():
    assert pick(W2, [1, 1], hdr(target="5")) == (None, "target_worker_miss")


def test_target_worker_miss_unhealthy():
    assert pick(W2, [1, 0], hdr(target="1")) == (None, "target_worker_miss")


def test_target_worker_priority_over_routing_key():
    assert pick(W2, [1, 1], hdr(target="1", key="some-key")) == (1, "target_worker_hit")


def test_fallback_random_distribution():
    dist = set()
    for i in range(100):
        idx, br = pick(W3, [1, 1, 1], None, seed=99, i=i)
        assert idx is not None and br == "random_fallback"
        dist.add(idx)
    assert len(dist) > 1


def test_no_healthy_workers():
    assert pick(["http://w1:8000"], [0], hdr(key="test")) == (None, "no_healthy_workers")


def test_empty_workers():
    assert pick([], [], None) == (None, "no_healthy_workers")


def test_consistent_hash_minimal_redistribution():
    urls = [f"http://w{i}:8000" for i in range(4)]
    ring = ch.Ring(urls)
    before = {i: pick(urls, [1, 1, 1, 1], hdr(key=f"user-{i}"), ring)[0] for i in range(100)}
    after = {i: pick(urls, [1, 0, 1, 1], hdr(key=f"user-{i}"), ring)[0] for i in range(100)}
    moved = sum(before[i] != after[i] for i in range(100))
    on_failed = sum(v == 1 for v in before.values())
    assert moved <= on_failed + 5 and moved < 50


def test_routing_key_failover_and_recovery():
    urls = [f"http://w{i}:8000" for i in range(3)]
    ring = ch.Ring(urls)
    orig, _ = pick(urls, [1, 1, 1], hdr(key="session-abc-123"), ring)
    healthy = [1, 1, 1]
    healthy[orig] = 0
    fail, _ = pick(urls, healthy, hdr(key="session-abc-123"), ring)
    assert fail != orig and healthy[fail]
    for _ in range(5):
        assert pick(urls, healthy, hdr(key="session-abc-123"), ring)[0] == fail
    assert pick(urls, [1, 1, 1], hdr(key="session-abc-123"), ring)[0] == orig


def test_empty_routing_key_uses_fallback():
    idx, br = pick(W2, [1, 1], hdr(key=""))
    assert idx is not None and br == "random_fallback"


def test_policy_name():
    from smg_b200 import ConsistentHashingPolicy
    assert ConsistentHashingPolicy.name(None) == "consistent_hashing"


# ---- hash_ring.rs tests ----
def test_ring_empty_returns_none():
    r = ch.Ring([])
    assert r.find_healthy_url(ch.key_position(b"any-key"), lambda u: True) is None
    assert len(ch.orc.HashRing([])) == 0 and ch.orc.HashRing([]).worker_count() == 0


def test_ring_len_scales_with_virtual_nodes():
    r = ch.orc.HashRing(["http://a", "http://b", "http://c"])
    assert len(r) == 450 and r.worker_count() == 3 and not r.is_empty()


def test_ring_find_healthy_url_is_deterministic_and_skips_unhealthy():
    r = ch.Ring(["http://a", "http://b", "http://c"])
    kp = ch.key_position(b"routing-key")
    first = r.find_healthy_url(kp, lambda u: True)
    assert all(r.find_healthy_url(kp, lambda u: True) == first for _ in range(10))
    assert r.find_healthy_url(kp, lambda u: u != "http://a") in ("http://b", "http://c")
    assert ch.Ring(["http://a", "http://b"]).find_healthy_url(ch.key_position(b"k"), lambda u: False) is None


def test_ring_agrees_with_oracle_ring_walk():
    urls = [f"http://w{i}:8000" for i in range(9)]
    r, o = ch.Ring(urls), ch.orc.HashRing(urls)
    for i in range(200):
        ok = lambda u, i=i: hash((u, i)) % 3 != 0   # noqa: E731
        key = f"k{i}"
        assert r.find_healthy_url(ch.key_position(key.encode()), ok) == o.find_healthy_url(key, ok)


# ---- the rules, one explicit case each ----
@pytest.mark.parametrize("value,expect", [("+3", 3), ("007", 7), (" 1", None), ("-0", None), ("+", None), ("18446744073709551615", None),
                                          ("18446744073709551616", None), ("3", 3), ("1a", None), ("++1", None)])
def test_target_parse(value, expect):
    urls = [f"http://w{i}:8000" for i in range(10)]
    idx, br = pick(urls, [1] * 10, hdr(target=value, key="k"))
    assert (idx, br) == ((expect, "target_worker_hit") if expect is not None else (None, "target_worker_miss"))
    assert ch.parse_usize(b"18446744073709551615") == 2**64 - 1   # parses; a miss only because it is ≥ len


def test_target_equal_to_len_misses():
    assert pick(W3, [1, 1, 1], hdr(target="3")) == (None, "target_worker_miss")


def test_target_ignores_circuit_breaker():
    # the oracle has no circuit breaker input: is_healthy() alone decides; the GPU test sets an open circuit on the same worker
    assert pick(W3, [1, 1, 1], hdr(target="2")) == (2, "target_worker_hit")


def test_non_visible_or_empty_target_falls_through_to_routing_key():
    want = pick(W3, [1, 1, 1], hdr(key="abc"))
    assert want[1] == "routing_key_hit"
    assert pick(W3, [1, 1, 1], hdr(target="é".encode(), key="abc")) == want
    assert pick(W3, [1, 1, 1], hdr(target="", key="abc")) == want
    assert pick(W3, [1, 1, 1], hdr(target=b"1\x7f", key="abc")) == want


def test_tab_is_visible():
    assert ch.to_str_ok(b"a\tb") and not ch.to_str_ok(b"a\nb") and not ch.to_str_ok(b"\x7f") and not ch.to_str_ok(b"\x80")


def test_empty_or_obs_text_authorization_does_not_fall_through():
    for auth in ("", "é".encode()):
        idx, br = pick(W3, [1, 1, 1], hdr(auth=auth, xff="10.0.0.1"))
        assert br == "random_fallback" and idx is not None
    # an absent authorization does fall through to x-forwarded-for, and an empty routing key falls through to authorization
    assert pick(W3, [1, 1, 1], hdr(xff="10.0.0.1"))[1] == "routing_key_hit"
    assert pick(W3, [1, 1, 1], hdr(key="", auth="Bearer t")) == pick(W3, [1, 1, 1], hdr(key="Bearer t"))
    assert pick(W3, [1, 1, 1], hdr(key="é".encode(), cookie="c=1")) == pick(W3, [1, 1, 1], hdr(key="c=1"))


def test_duplicate_urls_modulo_deduplicated_random_not():
    urls = ["http://a", "http://b", "http://a", "http://c"]
    view = ch.fleet_view(urls, [1, 1, 1, 1])
    assert view[1] == [1, 2, 3] and view[2] == [0, 1, 2, 3]
    for i in range(50):
        key = f"user-{i}".encode()
        assert pick(urls, [1, 1, 1, 1], hdr(key=key))[0] == [1, 2, 3][ch.key_position(key) % 3]
    seen = {pick(urls, [1, 1, 1, 1], None, seed=5, i=i)[0] for i in range(200)}
    assert seen == {0, 1, 2, 3}
    # the last HEALTHY index carries the URL
    assert ch.fleet_view(urls, [1, 1, 0, 1])[1] == [0, 1, 3]


def test_empty_ring_gives_none():
    assert pick(W3, [1, 1, 1], hdr(key="k"), ch.Ring([])) == (None, "no_healthy_workers")


def test_ring_urls_absent_from_slice():
    ring = ch.Ring(["http://x", "http://y"])
    assert pick(W3, [1, 1, 1], hdr(key="k"), ring) == (None, "no_healthy_workers")
    ring = ch.Ring(["http://x", "http://w2:8000"])
    for i in range(30):
        assert pick(W3, [1, 1, 1], hdr(key=f"k{i}"), ring) == (1, "routing_key_hit")


def test_headers_none_and_empty_slice_first():
    assert pick([], [], hdr(target="0")) == (None, "no_healthy_workers")
    assert pick(W3, [0, 0, 0], None) == (None, "no_healthy_workers")


def test_random_draw_maps_high_bits():
    seed = 12345
    for i in range(20):
        x = ch.draw(seed, i)
        assert pick(W3, [1, 0, 1], None, seed=seed, i=i)[0] == [0, 2][(x * 2) >> 64]


# ---- golden vectors (independent blake3) ----
def test_golden_key_positions():
    g = json.load(open(GOLDEN))
    assert len(g["keys"]) >= 20
    for k in g["keys"]:
        assert ch.key_position(gen.key_bytes(k["len"], k["salt"])) == int(k["pos"]), k["len"]


def test_golden_no_ring_decisions():
    g = json.load(open(GOLDEN))
    for d in g["no_ring_decisions"]:
        for r in d["requests"]:
            key = gen.key_bytes(r["len"], r["salt"])
            idx, br, kp = decide(d["urls"], d["healthy"], hdr(key=key), None, 0, 0)
            assert kp == int(r["pos"]) and (-1 if idx is None else idx) == r["idx"]
            assert br == ("routing_key_hit" if r["idx"] >= 0 else "no_healthy_workers")


# ---- HeaderValue::to_str on long values: a rejected byte at every residue mod 4 and at word-aligned middle offsets ----
@pytest.mark.parametrize("n", [9, 64, 1500])
def test_rejected_byte_anywhere_in_a_long_value(n):
    base = b"k" * n
    for at in sorted({0, 1, 2, 3, 4, 5, 6, 7, n // 2 - n // 2 % 4, n // 2 - n // 2 % 4 + 1, n - 4, n - 3, n - 2, n - 1}):
        for bad in (0x80, 0x01, 0x7F):
            v = base[:at] + bytes([bad]) + base[at + 1:]
            # a rejected target falls through to the routing key; a rejected implicit key goes to the random fallback
            assert pick(W3, [1, 1, 1], hdr(target=v, key="abc")) == pick(W3, [1, 1, 1], hdr(key="abc"))
            assert pick(W3, [1, 1, 1], hdr(cookie=v), seed=3, i=2) == pick(W3, [1, 1, 1], None, seed=3, i=2)
            assert pick(W3, [1, 1, 1], hdr(key=v, auth=base), ring=ch.Ring(W3)) == pick(W3, [1, 1, 1], hdr(key=base), ring=ch.Ring(W3))


# ---- the two restatements decide alike on seeded batches ----
def _random_headers(rng, n, w):
    hs = []
    for _ in range(n):
        if rng.random() < 0.05:
            hs.append(None)
            continue
        row = [None] * 5
        for h in range(5):
            if rng.random() < 0.35:
                u = rng.random()
                if h == 0 and u < 0.5:
                    row[h] = rng.choice([b"+1", b"007", b"-0", b"+", b"18446744073709551616", str(rng.randrange(w + 2)).encode()])
                else:
                    v = bytearray(gen.key_bytes(rng.choice([1, 9, 36, 200, 1024, 1025, 5000]), rng.randrange(1 << 30)))
                    if u > 0.8:
                        v[rng.randrange(len(v))] = rng.choice([0x80, 0x01, 0xFF])
                    row[h] = bytes(v) if u > 0.05 else b""
        hs.append(row)
    return hs


@pytest.mark.parametrize("w,ring_kind", [(1, "ring"), (3, "none"), (17, "ring"), (64, "empty"), (64, "partial")])
def test_python_and_cpp_restatements_agree(impl, w, ring_kind):
    if impl != "python":
        pytest.skip("one comparison covers both")
    import random
    rng = random.Random(w * 7 + len(ring_kind))
    urls = [f"http://worker-{i}:8000" if rng.random() > 0.1 else "http://dup:8000" for i in range(w)]
    healthy = [1 if rng.random() > 0.25 else 0 for _ in range(w)]
    ring_urls = {"ring": list(dict.fromkeys(urls)), "none": None, "empty": [], "partial": list(dict.fromkeys(urls))[:1] + ["http://x:1"]}[ring_kind]
    hs = _random_headers(rng, 1500, w)
    values, offs, present = ch.pack(hs, pad=3)
    oidx, obr, okp = ch.select_batch(urls, healthy, None if ring_urls is None else ch.Ring(ring_urls), hs, 99)
    for threads in (1, 4):
        idx, br, kp, _ = ch.cpp_select_batch(urls, healthy, ring_urls, values, offs, present, 99, threads)
        assert idx.tolist() == oidx and br == obr and kp.tolist() == okp
