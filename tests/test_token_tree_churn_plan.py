"""Colliding page keys and a churn plan for the token tree's device mirror (checked on CPU; replayed on the GPU by
tests/test_gpu_token_tree_churn.py).

The child key is page_finish(h1, h2, parent) with h1 = Σ (t_i + 1)·m1_i and h2 = Σ (t_i ^ 0x9E3779B9)·m2_i, both mod 2^32, and
every multiplier odd (smg_b200/csrc/token_tree.h).  Flipping bit 31 of one token changes each sum by 2^31·odd ≡ 2^31 (mod 2^32);
flipping it in an even number of the 16 positions changes neither sum.  So every page has 2^15 − 1 other pages with its key, under
every parent, and the host (`find_child`) and the kernel (the m == 0 branch of the probe loop) must compare labels, not keys.
This module restates the key, derives such families, and checks that the GPU tests' families really collide.  If the hash in
token_tree.h changes, `test_key_restatement_matches_token_tree_h` fails first: the families must then be derived again.

The plan is a seeded list of steps (batches, evictions, clears, new worker URLs) for the policy in token-tree mode.  `FlushModel`
says, from the oracle's node count before and after each step and the thresholds in token_tree.cu, which steps must reach the
device through the scatter kernel and which through a full re-upload; the CPU test asserts that the plan reaches every path:
growth of the initial 1024-slot table, an in-place rebuild, a full upload by eviction, and scatters."""
import itertools
import os
import re

import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE = 16
M32 = 0xFFFFFFFF
BIT31 = 0x80000000

# ---- thresholds of TokenTreeIndex (token_tree.cu) ----
TABLE0 = 1024          # slots of a new or cleared table
PATH_CAP = 32          # kPathCap: matched nodes the kernel reports
ROUND = 256            # tokens per label-compare round of the kernel
WINDOW = 512           # kWin: request tokens staged per warp


# =====================================================================================================================
# the page key, restated from token_tree.h
# =====================================================================================================================
def _mult1(i):
    x = ((i + 1) * 0x9E3779B9) & M32
    x ^= x >> 15
    x = (x * 0x85EBCA6B) & M32
    x ^= x >> 13
    return x | 1


def _mult2(i):
    x = ((i + 17) * 0xC2B2AE35) & M32
    x ^= x >> 16
    x = (x * 0x27D4EB2F) & M32
    x ^= x >> 14
    return x | 1


M1 = [_mult1(i) for i in range(PAGE)]
M2 = [_mult2(i) for i in range(PAGE)]


def page_finish(h1, h2, parent):
    a = h1 ^ ((parent * 0x85EBCA6B + 0xC2B2AE35) & M32)
    a ^= a >> 16; a = (a * 0x7FEB352D) & M32; a ^= a >> 15; a = (a * 0x846CA68B) & M32; a ^= a >> 16
    b = (h2 + parent * 0x27D4EB2F) & M32
    b ^= b >> 15; b = (b * 0x2C1B3C6D) & M32; b ^= b >> 12; b = (b * 0x297A2D39) & M32; b ^= b >> 15
    return ((a << 32) | b) | 1


def page_sums(page):
    h1 = sum(((int(t) + 1) & M32) * m for t, m in zip(page, M1)) & M32
    h2 = sum((int(t) ^ 0x9E3779B9) * m for t, m in zip(page, M2)) & M32
    return h1, h2


def page_key(page, parent):
    """key of (parent node id, first 16 tokens of the edge): page_key_host in token_tree.h"""
    assert len(page) == PAGE
    return page_finish(*page_sums(page), parent)


# the lines of token_tree.h the restatement above was written from
PINNED_HASH_LINES = [
    "__host__ __device__ inline uint32_t page_mult1(uint32_t i) { uint32_t x = (i + 1) * 0x9E3779B9u; x ^= x >> 15; x *= 0x85EBCA6Bu; x ^= x >> 13; return x | 1u; }",
    "__host__ __device__ inline uint32_t page_mult2(uint32_t i) { uint32_t x = (i + 17) * 0xC2B2AE35u; x ^= x >> 16; x *= 0x27D4EB2Fu; x ^= x >> 14; return x | 1u; }",
    "uint32_t a = h1 ^ (parent * 0x85EBCA6Bu + 0xC2B2AE35u);",
    "a ^= a >> 16; a *= 0x7FEB352Du; a ^= a >> 15; a *= 0x846CA68Bu; a ^= a >> 16;",
    "uint32_t b = h2 + parent * 0x27D4EB2Fu;",
    "b ^= b >> 15; b *= 0x2C1B3C6Du; b ^= b >> 12; b *= 0x297A2D39u; b ^= b >> 15;",
    "return (((uint64_t)a << 32) | b) | 1ULL;   // never 0 (0 marks an empty slot)",
    "for (uint32_t i = 0; i < kPage; ++i) { h1 += (page[i] + 1u) * M.m1[i]; h2 += (page[i] ^ 0x9E3779B9u) * M.m2[i]; }",
]
# the kernel's per-lane term: lanes 0-15 feed h1 with (t + 1) * m1, lanes 16-31 feed h2 with (t ^ 0x9E3779B9) * m2
PINNED_KERNEL_LINES = [
    "const uint32_t mult = rank < 16 ? page_mult1((uint32_t)rank) : page_mult2((uint32_t)rank - 16);",
    "const uint32_t salt_add = rank < 16 ? 1u : 0u, salt_xor = rank < 16 ? 0u : 0x9E3779B9u;",
    "const uint32_t term = ((t + salt_add) ^ salt_xor) * mult;",
]


# =====================================================================================================================
# collision families
# =====================================================================================================================
def flip_bit31(page, positions):
    p = np.array(page, dtype=np.uint32)
    for i in positions:
        p[i] ^= np.uint32(BIT31)
    return p


def even_subsets(positions=range(PAGE)):
    """the empty set, then every pair, then every quadruple of `positions`"""
    positions = list(positions)
    yield ()
    for k in range(2, len(positions) + 1, 2):
        yield from itertools.combinations(positions, k)


def collision_family(base, n, positions=range(PAGE)):
    """n distinct pages with `base`'s key under every parent: `base` with bit 31 flipped in an even set of `positions`"""
    out = [flip_bit31(base, s) for s in itertools.islice(even_subsets(positions), n)]
    assert len(out) == n, "not enough even subsets of these positions"
    return out


def straddling_page(rng):
    """a random page whose first tokens sit on both sides of 0x7FFFFFFF / 0x80000000, so that bit-31 flips reorder it against its
    siblings differently as u32 and as i32"""
    p = rng.integers(0, 1 << 32, size=PAGE, dtype=np.uint64).astype(np.uint32)
    p[:4] = [0x7FFFFFFF, 0x80000000, 0x7FFFFFFE, 0x80000001]
    return p


def fresh_page(rng):
    return rng.integers(0, 1 << 32, size=PAGE, dtype=np.uint64).astype(np.uint32)


def cat(*parts):
    parts = [np.asarray(p, dtype=np.uint32) for p in parts]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint32)


# the families the GPU tests use (seeded), so that they are checked here
def standalone_families():
    rng = np.random.default_rng(2024)
    return {
        "root64": collision_family(straddling_page(rng), 65),
        "tokens14_15": collision_family(straddling_page(rng), 2, positions=(14, 15)),
        "deep": collision_family(straddling_page(rng), 9),
        "evict": collision_family(straddling_page(rng), 25),
        "evict_under": collision_family(straddling_page(rng), 9),
    }


# =====================================================================================================================
# the churn plan for the policy in token-tree mode
# =====================================================================================================================
CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=16)
URLS0 = synth.worker_urls(6)
NEW_URLS = ["http://a-early:8000", "http://worker-00:8000"]   # sort before every URL of URLS0: the tenant ranks shift
PROBE = np.arange(5, dtype=np.uint32)                         # under one page: no walk, no touch, no insert


class Plan:
    """steps: ("batch", tag, requests, loads) | ("evict", max_size) | ("clear",) | ("urls", urls)"""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.steps = []
        self.shadow = orc.TokenTree()   # the node count of an insert-only stretch does not depend on the tenants
        self.n_workers = len(URLS0)
        self.fam_root = collision_family(straddling_page(self.rng), 12)
        self.fam_under = collision_family(straddling_page(self.rng), 8)
        self.fam_1415 = collision_family(straddling_page(self.rng), 2, positions=(14, 15))
        self.under = fresh_page(self.rng)                 # the ordinary page fam_under hangs below
        self.trunks = []
        self.seen = []

    def loads(self, imbalanced=False):
        l = self.rng.integers(0, 12, size=self.n_workers)
        if imbalanced:
            l[0] += 200
        return [int(x) for x in l]

    def tail(self, max_pages=4, ragged=True):
        k = int(self.rng.integers(0, max_pages + 1))
        n = PAGE * k + (int(self.rng.integers(0, PAGE)) if ragged and self.rng.random() < 0.3 else 0)
        return self.rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)

    def trunk(self):
        """a first page from a collision family (or an ordinary one), then ordinary pages"""
        r = self.rng.random()
        if r < 0.3:
            head = [self.fam_root[int(self.rng.integers(0, len(self.fam_root)))]]
        elif r < 0.55:
            head = [self.under, self.fam_under[int(self.rng.integers(0, len(self.fam_under)))]]
        elif r < 0.65:
            head = [self.fam_1415[int(self.rng.integers(0, 2))]]
        else:
            head = [fresh_page(self.rng)]
        return cat(*head, *[fresh_page(self.rng) for _ in range(int(self.rng.integers(0, 3)))])

    def request(self):
        if not self.trunks or self.rng.random() < 0.35:
            self.trunks.append(self.trunk())
        t = self.trunks[int(self.rng.integers(0, len(self.trunks)))]
        cut = len(t) if self.rng.random() < 0.7 else PAGE * int(self.rng.integers(1, len(t) // PAGE + 1))
        return cat(t[:cut], self.tail())

    def batch(self, tag, reqs, imbalanced=False, counted=False):
        for r in reqs if not counted else ():
            self.shadow.insert_tokens(r, "x")
        self.seen += reqs
        self.steps.append(("batch", tag, reqs, self.loads(imbalanced)))

    def replay_pair(self, collide):
        """two requests below a node T that ends exactly where both stop: the first inserts page P under T (or only a colliding
        sibling of P), the second walks T and stops at P.  Only the first kind invalidates the second request's snapshot walk."""
        T = cat(fresh_page(self.rng), fresh_page(self.rng))
        fam = collision_family(fresh_page(self.rng), 2, positions=(3, 11))
        self.batch("replay-base", [cat(T, fresh_page(self.rng)), cat(T, fresh_page(self.rng))])   # splits at |T|
        first = cat(T, fam[1] if collide else fam[0], fresh_page(self.rng))
        self.batch("replay-collide" if collide else "replay-same", [first, cat(T, fam[0], fresh_page(self.rng))])
        return T, fam

    def count(self):
        return self.shadow.node_count()


def churn_plan(seed=11):
    p = Plan(seed)
    # phase A: from an empty tree past 512 live children of the initial 1024-slot table, with scatters along the way
    p.batch("seed", [p.request() for _ in range(3)])
    p.replay_pair(collide=False)
    p.replay_pair(collide=True)
    k = 0
    while p.count() <= 560:
        k += 1
        if k == 6:
            p.steps.append(("urls", URLS0 + NEW_URLS))
            p.n_workers = len(URLS0) + len(NEW_URLS)
        if k % 3 == 0:
            p.batch(f"small{k}", [p.request() for _ in range(int(p.rng.integers(1, 3)))])
        else:
            p.batch(f"grow{k}", [p.request() for _ in range(int(p.rng.integers(10, 40)))], imbalanced=(k == 9))
    p.replay_pair(collide=True)
    p.steps.append(("evict", 900))
    p.batch("reinsert-a", [p.seen[int(i)] for i in p.rng.integers(0, len(p.seen), 30)] + [p.request() for _ in range(10)])
    p.steps.append(("evict", 16))
    p.batch("reinsert-b", [cat(f, fresh_page(p.rng)) for f in p.fam_root[::2]] + [p.request() for _ in range(10)])
    p.steps.append(("clear",))
    # phase B: exactly 512 live nodes with no tombstone, then an eviction to few live nodes, then inserts: an in-place rebuild
    p.shadow.clear()
    k = 0
    while p.count() < 500:
        k += 1
        reqs = []
        for _ in range(int(p.rng.integers(1, 30)) if k % 4 else 1):
            if p.count() >= 500:
                break
            reqs.append(p.request())
            p.shadow.insert_tokens(reqs[-1], "x")   # a request adds at most 3 nodes: this stops at 500-502
        p.batch(f"refill{k}", reqs, counted=True)
    pad = []
    while p.count() + len(pad) < 512:
        pad.append(cat(fresh_page(p.rng), p.tail(2, ragged=False)))   # one new leaf under the root each
    p.batch("pad-to-512", pad)
    assert p.count() == 512
    p.steps.append(("evict", 32))
    p.batch("rebuild-in-place", [p.request() for _ in range(12)])
    p.batch("small-after-rebuild", [p.request()])
    p.replay_pair(collide=False)
    p.steps.append(("evict", 256))
    p.batch("reinsert-c", [p.seen[int(i)] for i in p.rng.integers(0, len(p.seen), 20)], imbalanced=True)
    p.steps.append(("urls", URLS0 + NEW_URLS + ["http://0-first:8000"]))
    p.n_workers += 1
    p.batch("after-urls", [p.request() for _ in range(15)])
    return p


def _next_pow2(x):
    return 1 << max(0, int(x - 1).bit_length())


class FlushModel:
    """What TokenTreeIndex::flush does with the dirt of one plan step, from node counts alone.

    Within a clean stretch (no eviction since the start or the last clear) node ids are allocated contiguously, the table has no
    tombstone, nodes_ has 1 + live entries and its capacity only doubles.  Then:
      * a step that stays at ≤ 512 live nodes does not rebuild the 1024-slot table ((live + tombs + 1)·2 > size only from 512);
      * it does not grow nodes_ (which forces a full upload) while 1 + live stays within the capacity the stretch reached;
      * a batch of r requests of p pages dirties at most Σ (2p + 4) slots: touched nodes, one split, its re-keyed child, a leaf.
      If that is ≤ 1024 / 8, flush scatters.
    Full uploads that are certain: a clear; a batch that passes 512 live nodes in a clean stretch (table rebuild); an eviction
    that removes more than cap/8 nodes, cap bounded by the smallest 1024·2^k ≥ 4·(peak since the clear); the first inserting batch
    after an eviction that left live + tombs ≥ 512 (the table rebuilds: in place when (live + 1)·4 ≤ 1024).  A batch's full upload
    is only certain at the next flush in SNAPSHOT mode: in SEQUENTIAL mode a restart may flush it mid-batch, and the requests after
    the restart then leave a few dirty slots.
    `step` returns "scatter", "full" or None (not decided by counts)."""

    def __init__(self, snapshot):
        self.snapshot = snapshot
        self.clean = True
        self.peak = 0            # peak live nodes since the last clear
        self.cap_vec = 1         # capacity of nodes_ (exact while clean since the start, a lower bound after a clear)
        self.sum_at_evict = None   # live + tombs right after the first eviction of a clean stretch (exact)
        self.inplace = 0
        self.growth = 0

    def step(self, step, c0, c1):
        kind = step[0]
        out = None
        if kind == "clear":
            self.clean, self.peak, self.sum_at_evict = True, 0, None
            return "full"
        if kind == "urls":
            return None
        if kind == "evict":
            cap_max = TABLE0
            while cap_max < 4 * self.peak:
                cap_max *= 2
            if c0 - c1 > cap_max // 8:
                out = "full"
            self.sum_at_evict = c0 if (self.clean and c0 <= 512) else None   # the table still has its 1024 slots
            self.clean = False
            return out
        reqs = step[2]
        if self.clean:
            dirty = sum(2 * (len(r) // PAGE) + 4 for r in reqs)
            if c0 <= 512 < c1:                          # the insert that finds 512 live nodes rebuilds the 1024-slot table
                out = "full" if self.snapshot else None
                self.growth += 1
            elif c0 > 512:
                pass
            elif 1 + c1 <= self.cap_vec and dirty <= TABLE0 // 8 and any(len(r) >= PAGE for r in reqs):
                out = "scatter"
            self.cap_vec = max(self.cap_vec, _next_pow2(1 + c1))
        elif self.sum_at_evict is not None:
            if self.sum_at_evict >= 512 and c1 > c0:   # the first new node finds (live + tombs + 1)·2 > 1024
                out = "full" if self.snapshot else None
                self.inplace += (c0 + 1) * 4 <= TABLE0
            self.sum_at_evict = None
        self.peak = max(self.peak, c0, c1)
        return out


# =====================================================================================================================
# CPU tests
# =====================================================================================================================
def test_key_restatement_matches_token_tree_h():
    """the restated key is the one in token_tree.h and token_tree.cu — if this fails, the hash changed: restate it and derive the
    collision families again, or the GPU collision tests stop testing collisions"""
    def norm(s):
        return re.sub(r"\s+", " ", s).strip()
    with open(os.path.join(ROOT, "smg_b200", "csrc", "token_tree.h")) as f:
        h = norm(f.read())
    with open(os.path.join(ROOT, "smg_b200", "csrc", "token_tree.cu")) as f:
        cu = norm(f.read())
    for line in PINNED_HASH_LINES:
        assert norm(line) in h, f"page hash in token_tree.h changed: {line}"
    for line in PINNED_KERNEL_LINES:
        assert norm(line) in cu, f"page hash in tree_walk_request changed: {line}"


def test_restated_key_known_answers():
    """the restated multipliers are odd and distinct, and the key is never 0 — the properties the collision argument uses"""
    assert all(m & 1 for m in M1 + M2)
    assert len(set(M1)) == PAGE and len(set(M2)) == PAGE
    rng = np.random.default_rng(3)
    for _ in range(200):
        assert page_key(fresh_page(rng), int(rng.integers(0, 1 << 32))) != 0
    # a single flipped bit 31 moves both sums by exactly 2^31, so such pages do NOT collide
    p = fresh_page(rng)
    h1, h2 = page_sums(p)
    for i in range(PAGE):
        g1, g2 = page_sums(flip_bit31(p, [i]))
        assert (g1 ^ h1, g2 ^ h2) == (BIT31, BIT31)
        assert page_key(flip_bit31(p, [i]), 0) != page_key(p, 0)


def _plan_parents(plan):
    """node ids the plan's trees can reach: a tree never holds more nodes than the tokens it saw have pages, plus the root"""
    return range(0, 2 * sum(len(r) // PAGE for s in plan.steps if s[0] == "batch" for r in s[2]) + 2, 97)


def test_families_collide():
    """every family the GPU tests use: distinct pages, one key each under the root, deep parents and the plan's node ids"""
    plan = churn_plan()
    fams = dict(standalone_families())
    fams.update(plan_root=plan.fam_root, plan_under=plan.fam_under, plan_1415=plan.fam_1415)
    parents = list(range(0, 130)) + list(_plan_parents(plan)) + [0xFFFFFFFD]
    for name, fam in fams.items():
        assert len({tuple(int(x) for x in m) for m in fam}) == len(fam), name
        sums = {page_sums(m) for m in fam}
        assert len(sums) == 1, name
        for parent in parents:
            assert len({page_key(m, parent) for m in fam}) == 1, (name, parent)
        assert any(int(t) >= BIT31 for m in fam for t in m) and any(int(t) < BIT31 for m in fam for t in m), name
    # tokens 14 and 15: the members agree on 0..13, so a label compare reaches token 14 before it differs
    a, b = fams["tokens14_15"]
    assert (a[:14] == b[:14]).all() and (a[14:] != b[14:]).all()


def _replay_oracle(plan, mode):
    """the plan on the oracle policy → per step (kind, node count before, after, flush expectation, decisions)"""
    orc.reset_globals()
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **CFG)
    urls = list(URLS0)
    op.set_workers(urls)
    op.set_state([0] * len(urls), [1] * len(urls), [1] * len(urls))
    fm = FlushModel(mode == "snapshot")
    rows = []
    for st in plan.steps:
        c0 = op.token_tree().node_count()
        dec = None
        if st[0] == "batch":
            op.set_state(st[3], [1] * len(st[3]), [1] * len(st[3]))
            if mode == "snapshot":
                off = np.zeros(len(st[2]) + 1, np.uint64)
                np.cumsum([len(r) for r in st[2]], out=off[1:])
                _, br, ma, _ = op.select_batch_tokens(cat(*st[2]), off, snapshot=True)
                dec = [(orc.BRANCHES[int(b)], int(m)) for b, m in zip(br, ma)]
            else:
                dec = [(d.branch, d.matched) for d in (op.select_worker(tokens=r) for r in st[2])]
        elif st[0] == "evict":
            op.evict_cache(st[1])
        elif st[0] == "clear":
            op.token_tree().clear()
        elif st[0] == "urls":
            urls = list(st[1])
            op.set_workers(urls)
        c1 = op.token_tree().node_count()
        rows.append((st, c0, c1, fm.step(st, c0, c1), dec))
    return rows, fm


@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
def test_plan_reaches_every_flush_path(mode):
    plan = churn_plan()
    rows, fm = _replay_oracle(plan, mode)
    kinds = [r[0][0] for r in rows]
    assert {"batch", "evict", "clear", "urls"} <= set(kinds)
    # growth: past 512 live children of the initial 1024-slot table, in a stretch without tombstones
    assert fm.growth >= 1
    # eviction of more than 1/8 of the table's slots in one step
    assert any(r[0][0] == "evict" and r[3] == "full" for r in rows)
    # scatters: several batches whose few dirty slots flush through the scatter kernel
    assert sum(r[3] == "scatter" for r in rows) >= 4
    # an in-place rebuild: exactly 512 live nodes without tombstones, an eviction to ≤ 255, then an inserting batch
    i = next(i for i, r in enumerate(rows) if r[0][0] == "batch" and r[0][1] == "pad-to-512")
    assert rows[i][2] == 512
    assert rows[i + 1][0] == ("evict", 32) and rows[i + 1][2] <= 255
    assert rows[i + 2][3] == ("full" if mode == "snapshot" else None) and rows[i + 2][2] > rows[i + 2][1]
    assert fm.inplace >= 1
    # a mix of branches, and collision families under the root and below a node
    branches = {b for r in rows if r[4] for b, _ in r[4]}
    assert {"tree_match", "tree_min_load", "imbalanced_min_load"} <= branches


@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
def test_replay_pairs_stop_where_intended(mode):
    """in "replay-same" the first request inserts the page the second stops at, so the second matches one page further than the
    node T; in "replay-collide" it inserts only a colliding sibling, and the second still matches |T| = 32 tokens"""
    rows, _ = _replay_oracle(churn_plan(), mode)
    same = [r for r in rows if r[0][0] == "batch" and r[0][1] == "replay-same"]
    coll = [r for r in rows if r[0][0] == "batch" and r[0][1] == "replay-collide"]
    assert same and coll
    for r in same:
        assert r[4][1][1] == (32 if mode == "snapshot" else 48), r[4]
    for r in coll:
        assert r[4][1][1] == 32, r[4]
