"""CPU restatement of ConsistentHashingPolicy (model_gateway/src/policies/consistent_hashing.rs:116-186) — test infrastructure only.

Rules, line by line:
  1. an empty worker slice → (None, no_healthy_workers) before any header is read (:121-123);
  2. extract_header_value (routers/common/header_utils.rs:60-65): HeaderMap::get (the first value) → HeaderValue::to_str (every byte
     is \\t or 0x20..=0x7E) → non-empty;
  3. X-SMG-Target-Worker, if extracted: usize::from_str (64-bit: optional '+', one or more ASCII digits, overflow is an error); a hit
     needs idx < len and is_healthy(), anything else is (None, target_worker_miss) (:128-137);
  4. X-SMG-Routing-Key, if extracted: find_by_consistent_hash → routing_key_hit, or (None, no_healthy_workers) (:139-145);
  5. the implicit key: the first PRESENT of authorization, x-forwarded-for, cookie, then to_str and the non-empty filter (:147-161);
  6. find_by_consistent_hash (:68-111): url → LAST healthy slice index (circuit breaker not read); empty map → None; with a ring,
     HashRing::find_healthy_url (blake3(key)[..8] LE, partition_point, clockwise walk); without one, the sorted map values indexed by
     u64_le(blake3(key)[..8]) % len;
  7. the random fallback (:163-185): healthy_count over every is_healthy() worker (duplicates included), 0 → no_healthy_workers, else
     the random_range(0..healthy_count)-th healthy worker.  rand::rng() cannot be seeded, so request i of a batch uses draw i of the
     power_of_two counter stream: x = splitmix64-finalise(seed + GOLDEN·(i + 1)), index ⌊x·h / 2^64⌋.
blake3 is the oracle's own restatement (oracle/blake3_ref.h through orc.blake3_digest); the ring is orc.HashRing.
The C++ restatement (tests/cpp/consistent_hashing_oracle.h, built as tests/cpp/libchash_oracle.so) is driven by cpp_select_batch; the CPU
tests hold the two to the same decisions.
"""
import bisect
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import orc

CPP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")
_cpp = None

HEADERS = ("x-smg-target-worker", "x-smg-routing-key", "authorization", "x-forwarded-for", "cookie")
BRANCHES = ("no_healthy_workers", "target_worker_hit", "target_worker_miss", "routing_key_hit", "random_fallback")
M64 = 2**64 - 1


def finalise(x):
    x ^= x >> 30; x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27; x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def draw(seed, k):
    """Draw k (0-based) of the stream `seed`."""
    return finalise((seed + 0x9E3779B97F4A7C15 * (k + 1)) & M64)


def key_position(key: bytes) -> int:
    """u64::from_le_bytes(blake3(key)[..8]) (hash_ring.rs:78-86, consistent_hashing.rs:98-108)."""
    return int.from_bytes(orc.blake3_digest(key)[:8], "little")


def to_str_ok(v: bytes) -> bool:
    return all(c == 9 or 0x20 <= c <= 0x7E for c in v)


def extract(v):
    return v if v is not None and to_str_ok(v) and len(v) else None


def parse_usize(v: bytes):
    s = v[1:] if v[:1] == b"+" else v
    if not s or any(not 0x30 <= c <= 0x39 for c in s):
        return None
    x = int(s)
    return x if x <= M64 else None


class Ring:
    """The sorted (position, URL) entries of an orc.HashRing, walked as find_healthy_url does."""

    def __init__(self, urls):
        self.urls = list(urls)
        pos, url = orc.HashRing(self.urls).entries()
        self.pos = [int(p) for p in pos]
        self.url = [self.urls[int(u)] for u in url]

    def find_healthy_url(self, key_pos, is_healthy):
        n = len(self.pos)
        if n == 0:
            return None
        start = bisect.bisect_left(self.pos, key_pos)   # partition_point(|pos| pos < key_pos)
        for i in range(n):
            u = self.url[(start + i) % n]
            if is_healthy(u):
                return u
        return None


def fleet_view(urls, healthy):
    """What select_worker_impl derives from the slice: healthy_url_to_idx (collect(): a later duplicate URL overwrites) and the
    is_healthy() indices in slice order.  Computed once per batch: every request of a batch reads one fleet snapshot."""
    url_to_idx = {}
    for i, u in enumerate(urls):
        if healthy[i]:
            url_to_idx[u] = i
    return url_to_idx, sorted(url_to_idx.values()), [j for j in range(len(urls)) if healthy[j]]


def find_by_consistent_hash(view, ring, key: bytes):
    """→ (idx or None, key position)."""
    url_to_idx, vals, _ = view
    kp = key_position(key)
    if not url_to_idx:
        return None, kp
    if ring is not None:
        u = ring.find_healthy_url(kp, lambda x: x in url_to_idx)
        return (None if u is None else url_to_idx[u]), kp
    return vals[kp % len(vals)], kp


def select_worker(urls, healthy, ring, headers, seed, i, view=None):
    """One request.  headers: five values (bytes, or None when HeaderMap::get returns None) in HEADERS order, or None for
    info.headers = None.  → (idx or None, branch name, key position or 0)."""
    if not urls:
        return None, "no_healthy_workers", 0
    view = view or fleet_view(urls, healthy)
    hv = list(headers) if headers is not None else [None] * 5
    target = extract(hv[0])
    if target is not None:
        t = parse_usize(target)
        if t is not None and t < len(urls) and healthy[t]:
            return t, "target_worker_hit", 0
        return None, "target_worker_miss", 0
    key = extract(hv[1])
    if key is None:
        first = next((v for v in hv[2:5] if v is not None), None)
        key = extract(first)
    if key is not None:
        idx, kp = find_by_consistent_hash(view, ring, key)
        return idx, ("routing_key_hit" if idx is not None else "no_healthy_workers"), kp
    hs = view[2]
    if not hs:
        return None, "no_healthy_workers", 0
    return hs[(draw(seed, i) * len(hs)) >> 64], "random_fallback", 0


def select_batch(urls, healthy, ring, headers_list, seed):
    """Request i uses draw i of `seed`.  → (idx list with -1 for None, branch names, key positions)."""
    out, br, kps = [], [], []
    view = fleet_view(urls, healthy)
    for i, h in enumerate(headers_list):
        idx, b, kp = select_worker(urls, healthy, ring, h, seed, i, view)
        out.append(-1 if idx is None else idx)
        br.append(b)
        kps.append(kp)
    return out, br, kps


def _cpp_lib():
    global _cpp
    if _cpp is None:
        subprocess.check_call(["make", "-s", "-C", CPP, "-f", "consistent_hashing.mk", "libchash_oracle.so"])
        L = C.CDLL(os.path.join(CPP, "libchash_oracle.so"))
        L.chorc_ring_new.restype = C.c_void_p
        L.chorc_ring_new.argtypes = [C.POINTER(C.c_char_p), C.c_size_t]
        L.chorc_ring_free.argtypes = [C.c_void_p]
        L.chorc_select_batch.restype = C.c_double
        L.chorc_select_batch.argtypes = [C.POINTER(C.c_char_p), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                         C.c_uint64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _cpp = L
    return _cpp


def pack(headers_list, pad=0):
    """The packed form of smgx_consistent_hashing_select_batch: values, 5n + 1 offsets (starting at `pad`), presence masks."""
    blob, offs, present = bytearray(b"\x00" * pad), [pad], []
    for row in headers_list:
        bits = 0
        for h in range(5):
            v = None if row is None else row[h]
            if v is not None:
                bits |= 1 << h
                blob += v
            offs.append(len(blob))
        present.append(bits)
    return bytes(blob), offs, present


def cpp_select_batch(urls, healthy, ring_urls, values, offsets, present, seed, threads=1):
    """The C++ oracle on `threads` host threads; ring_urls None = no ring.  → (idx int32[n], branch names, key positions uint64[n], seconds)."""
    L = _cpp_lib()
    enc = [u.encode() for u in urls]
    arr = (C.c_char_p * max(len(enc), 1))(*enc)
    hl = np.ascontiguousarray(np.asarray(list(healthy) or [0], np.uint8))
    ring = None
    if ring_urls is not None:
        renc = [u.encode() for u in ring_urls]
        ring = L.chorc_ring_new((C.c_char_p * max(len(renc), 1))(*renc), len(renc))
    vb = np.frombuffer(values, np.uint8) if len(values) else np.zeros(1, np.uint8)
    off = np.ascontiguousarray(np.asarray(offsets, np.uint32))
    pr = np.ascontiguousarray(np.asarray(present, np.uint8))
    n = pr.size
    idx, br, kp = np.full(max(n, 1), -1, np.int32), np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.uint64)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    try:
        secs = L.chorc_select_batch(arr, ptr(hl), len(urls), ring, ptr(vb), ptr(off), ptr(pr), n, seed & M64, threads, ptr(idx), ptr(br), ptr(kp))
    finally:
        if ring:
            L.chorc_ring_free(ring)
    return idx[:n], [BRANCHES[b] for b in br[:n]], kp[:n], secs
