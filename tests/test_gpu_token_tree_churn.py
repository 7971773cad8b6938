"""The token tree's device mirror under colliding page keys, token ids of 2^31 and above, and churn (eviction, node reuse, table
rebuilds, clears, new tenants), against the oracle: `orc.TokenTree` for the standalone tree, `orc.CacheAwarePolicy` for the policy
in token-tree mode.  The families and the plan come from tests/test_token_tree_churn_plan.py, which checks on CPU that the families
collide and that the plan reaches every flush path."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc
from tests import test_token_tree_churn_plan as P

pytestmark = pytest.mark.gpu

PAGE = P.PAGE
TENANTS = ["t-a", "t-b", "t-c"]


def _trees(policy):
    from smg_b200 import TokenTree
    t = TokenTree.standalone(policy)
    orc.reset_globals()
    return t, orc.TokenTree(policy)


def _check(t, o, queries, tag):
    """every query matched by the GPU walk and the oracle; then the whole tree (timestamps included) and the per-tenant sizes"""
    for i, q in enumerate(queries):
        g, w = t.match_prefix_with_counts(q), o.match_prefix_with_counts(q)
        assert (g.matched_token_count, g.input_token_count, g.tenant) == (w.matched_token_count, w.input_token_count, w.tenant), (tag, i)
    assert t.entries() == o.entries(), tag
    for ten in TENANTS:
        assert t.tenant_token_size(ten) == o.tenant_token_size(ten), (tag, ten)


def _insert(t, o, seq, tenant):
    t.insert_tokens(seq, tenant)
    o.insert_tokens(seq, tenant)


def _family_queries(prefix, fam, exts, absent):
    cat = P.cat
    q = []
    for m, e in zip(fam, exts):
        q += [cat(prefix, m), cat(prefix, m, e), cat(prefix, m, e, e[:7]), cat(prefix, m, e[::-1])]
    q += [cat(prefix, absent), cat(prefix, absent, exts[0])]
    return q


def _build_family(t, o, prefix, fam, exts, rng):
    """members inserted in several orders by several tenants: t-a each member with its extension, t-b each member alone in reverse
    order (splits), t-c every third member in a shuffled order"""
    for m, e in zip(fam, exts):
        _insert(t, o, P.cat(prefix, m, e), "t-a")
    for m in fam[::-1]:
        _insert(t, o, P.cat(prefix, m), "t-b")
    for i in rng.permutation(len(fam))[::3]:
        _insert(t, o, P.cat(prefix, fam[i], exts[i], exts[(i + 1) % len(fam)]), "t-c")


@pytest.mark.parametrize("n", [2, 3, 16, 64])
def test_collision_family_under_root(n):
    """n pages with one key under the root: every member, every member extended, and a member never inserted, which must walk the
    whole probe chain and match 0"""
    fam = P.standalone_families()["root64"]
    rng = np.random.default_rng(n)
    members, absent = fam[:n], fam[64]
    exts = [P.fresh_page(rng) for _ in members]
    t, o = _trees(0)
    _build_family(t, o, P.cat(), members, exts, rng)
    assert o.node_count() >= n                          # n distinct children of the root, one key
    qs = _family_queries(P.cat(), members, exts, absent)
    _check(t, o, qs, "root")
    assert t.match_prefix_with_counts(absent).matched_token_count == 0
    for m in members:
        assert t.match_prefix_with_counts(m).matched_token_count == PAGE


def test_collision_in_tokens_14_and_15():
    """two members equal in tokens 0-13: the label compare stops at token 14 and rounds down to m = 0, so the walk must keep probing"""
    a, b = P.standalone_families()["tokens14_15"]
    rng = np.random.default_rng(5)
    e = P.fresh_page(rng)
    for first, second in ((a, b), (b, a)):
        t, o = _trees(0)
        _insert(t, o, P.cat(first, e), "t-a")
        _check(t, o, [first, second, P.cat(second, e)], "one")
        assert t.match_prefix_with_counts(second).matched_token_count == 0
        _insert(t, o, P.cat(second, e), "t-b")
        _insert(t, o, P.cat(e, second), "t-c")          # the pair again below a node
        _insert(t, o, P.cat(e, first, e), "t-a")
        _check(t, o, [first, second, P.cat(first, e), P.cat(second, e), P.cat(e, first), P.cat(e, second, e), P.cat(e, first, e, e)], "two")


def _deep_prefix(t, o, where, rng):
    """a prefix that ends at a node boundary; the family hangs below it"""
    if where == "page2":
        prefix = P.fresh_page(rng)
    elif where == "after_round":
        prefix = P.cat(*[P.fresh_page(rng) for _ in range(P.ROUND // PAGE)])
    elif where == "after_window":
        prefix = P.cat(*[P.fresh_page(rng) for _ in range(P.WINDOW // PAGE)])
    else:   # past the 32-node path cap: a chain of 36 nodes, one page each
        prefix = P.cat(*[P.fresh_page(rng) for _ in range(36)])
        for k in range(36, 0, -1):
            _insert(t, o, prefix[: k * PAGE], "t-c")
    return prefix


@pytest.mark.parametrize("where", ["page2", "past_path_cap", "after_round", "after_window"])
def test_collision_family_below_deep_nodes(where):
    fam = P.standalone_families()["deep"]
    members, absent = fam[:8], fam[8]
    rng = np.random.default_rng(len(where))
    t, o = _trees(0)
    prefix = _deep_prefix(t, o, where, rng)
    exts = [P.fresh_page(rng) for _ in members]
    _build_family(t, o, prefix, members, exts, rng)
    qs = _family_queries(prefix, members, exts, absent)
    _check(t, o, qs, where)
    for m, e in zip(members, exts):
        assert t.match_prefix_with_counts(P.cat(prefix, m, e)).matched_token_count == len(prefix) + 2 * PAGE
    assert t.match_prefix_with_counts(P.cat(prefix, absent)).matched_token_count == len(prefix)


@pytest.mark.parametrize("policy", range(6), ids=["lru", "lfu", "fifo", "mru", "filo", "priority"])
def test_eviction_leaves_tombstones_in_collision_chains(policy):
    """evict members of two families (under the root and below a node) so that tombstones sit inside their probe chains; match
    survivors and evicted members; reinsert onto the tombstones (reusing freed node ids); evict by size; clear and rebuild"""
    fams = P.standalone_families()
    root, under = fams["evict"][:24], fams["evict_under"][:8]
    rng = np.random.default_rng(100 + policy)
    node = P.fresh_page(rng)
    t, o = _trees(policy)
    exts_r = [P.fresh_page(rng) for _ in root]
    exts_u = [P.fresh_page(rng) for _ in under]
    seqs = [P.cat(m, e) for m, e in zip(root, exts_r)] + [P.cat(node, m, e) for m, e in zip(under, exts_u)]
    for i, s in enumerate(seqs):                        # t-a owns all; t-b every third; t-c every fifth (different orders)
        _insert(t, o, s, "t-a")
    for s in seqs[::-3]:
        _insert(t, o, s, "t-b")
    for s in seqs[1::5]:
        _insert(t, o, s[:PAGE] if len(s) == 2 * PAGE else s[: 2 * PAGE], "t-c")
    qs = _family_queries(P.cat(), root, exts_r, fams["evict"][24]) + _family_queries(node, under, exts_u, fams["evict_under"][8])
    _check(t, o, qs, "built")
    # interleave matches so that the policies' orders differ from insertion order
    for s in seqs[5::4]:
        t.match_prefix_with_counts(s); o.match_prefix_with_counts(s)
    n0 = o.node_count()
    t.evict_tenant("t-a", t.tenant_token_size("t-a") // 2)
    o.evict_tenant("t-a", o.tenant_token_size("t-a") // 2)
    assert o.node_count() < n0                          # slots were tombstoned
    _check(t, o, qs, "evicted-a")
    t.evict_tenant("t-b", PAGE)
    o.evict_tenant("t-b", PAGE)
    _check(t, o, qs, "evicted-b")
    for s in seqs[::2]:                                 # reinsert: table_insert takes the first tombstone of each chain
        _insert(t, o, s, "t-b")
    for s in seqs[1::6]:
        _insert(t, o, P.cat(s, P.fresh_page(rng)), "t-c")
    _check(t, o, qs, "reinserted")
    t.evict_tenant_by_size(3 * PAGE)
    o.evict_tenant_by_size(3 * PAGE)
    _check(t, o, qs, "by-size")
    t.clear(); o.clear()
    _check(t, o, qs, "cleared")
    for s in seqs[::-1]:
        _insert(t, o, s, "t-c")
    _check(t, o, qs, "after-clear")


def test_entries_order_across_bit31():
    """siblings whose first tokens straddle 0x7FFFFFFF / 0x80000000: entries() and eviction order them as unsigned 32-bit ids"""
    rng = np.random.default_rng(9)
    base = P.straddling_page(rng)
    pages = [base] + [P.flip_bit31(base, [i]) for i in range(4)] + [P.flip_bit31(base, [0, 1]), P.flip_bit31(base, [2, 3])]
    for policy in (0, 2, 4):
        t, o = _trees(policy)
        for k, pg in enumerate(pages):
            _insert(t, o, P.cat(pg, P.fresh_page(rng)), "t-a")
            _insert(t, o, pg, TENANTS[k % 3])
        _check(t, o, pages, "built")
        ents = t.entries()
        firsts = [tuple(e[0][:PAGE]) for e in ents if len(e[0]) == PAGE]
        assert firsts == sorted(firsts)                 # Python ints: unsigned order
        t.evict_tenant("t-a", 3 * 2 * PAGE); o.evict_tenant("t-a", 3 * 2 * PAGE)
        _check(t, o, pages, "evicted")


def test_insert_after_eviction_restores_the_root_tenant():
    """known answer: eviction that empties a tenant's subtree also removes it from the root; the tenant's next insert puts it back
    at the root (token_tree.rs:412-416 does so on every insert), not only its first insert"""
    rng = np.random.default_rng(21)
    a, b = P.cat(P.fresh_page(rng), P.fresh_page(rng)), P.cat(P.fresh_page(rng))
    t, o = _trees(0)
    _insert(t, o, a, "t-a")
    _insert(t, o, a, "t-a")                            # the count is inflated to 64 (:467-474): eviction goes on to the root
    _insert(t, o, b, "t-b")
    t.evict_tenant("t-a", 0); o.evict_tenant("t-a", 0)
    _check(t, o, [a, b], "evicted")
    assert [x for x, _ in t.entries()[0][1]] == ["t-b"]
    _insert(t, o, b, "t-a")
    _check(t, o, [a, b], "reinserted")
    assert t.entries()[0] == ([], [("t-a", 0), ("t-b", 0)])


# =====================================================================================================================
# the policy in token-tree mode through the churn plan
# =====================================================================================================================
def _policy_pair(mode):
    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **P.CFG), tree_batch_mode=mode)
    ws = [BasicWorker(u) for u in P.URLS0]
    pol.init_workers(ws)
    orc.reset_globals()
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **P.CFG)
    op.set_workers(list(P.URLS0))
    return pol, ws, op


def _set_fleet(ws, op, loads):
    for w, l in zip(ws, loads):
        w.set_load(int(l)); w.set_healthy(True)
    op.set_state(loads, [1] * len(ws), [1] * len(ws))


def _route(pol, ws, op, reqs, mode, tag):
    idx, info = pol.select_worker_batch(ws, reqs)
    if mode == "snapshot":
        off = np.zeros(len(reqs) + 1, np.uint64)
        np.cumsum([len(r) for r in reqs], out=off[1:])
        want, br, ma, _ = op.select_batch_tokens(P.cat(*reqs), off, snapshot=True)
        for i in range(len(reqs)):
            assert (want[i], br[i], ma[i], len(reqs[i])) == (idx[i], info[i].branch, info[i].matched, info[i].input), (tag, i)
    else:
        for i, r in enumerate(reqs):
            d = op.select_worker(tokens=r)
            assert (d.idx if d.idx is not None else -1) == idx[i], (tag, i, d.branch, orc.BRANCHES[info[i].branch])
            assert (d.branch, d.matched, d.input) == (orc.BRANCHES[info[i].branch], info[i].matched, info[i].input), (tag, i)
    return idx, info


def _probe(pol, ws, op, mode, tag):
    """two selects of one request shorter than a page (no walk, no touch, no insert) on the same fleet: they launch the same
    kernels except that only the first flushes the mirror.  → scatter kernels the first one ran"""
    a = pol.kernel_launches()
    _route(pol, ws, op, [P.PROBE], mode, tag)
    b = pol.kernel_launches()
    _route(pol, ws, op, [P.PROBE], mode, tag)
    c = pol.kernel_launches()
    return (b - a) - (c - b)


def _same_state(pol, op, urls, tag):
    assert pol.token_tree().entries() == op.token_tree().entries(), tag
    for u in urls:
        assert pol.token_tree().tenant_token_size(u) == op.token_tree().tenant_token_size(u), (tag, u)


@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
def test_churn_plan_policy(mode):
    """every decision of the plan equals the oracle's; after every step the trees (timestamps included) and the tenant sizes are
    equal; the steps the flush model decides go through the scatter kernel or a full upload as it says; at the end the device walk
    entry point over all the plan's requests equals one oracle snapshot call"""
    from smg_b200 import BasicWorker
    plan = P.churn_plan()
    pol, ws, op = _policy_pair(mode)
    urls = list(P.URLS0)
    loads = [0] * len(urls)
    _set_fleet(ws, op, loads)
    fm = P.FlushModel(mode == "snapshot")
    seen = {"scatter": 0, "full": 0}
    for k, st in enumerate(plan.steps):
        c0 = op.token_tree().node_count()
        if st[0] == "batch":
            loads = st[3]
            _set_fleet(ws, op, loads)
            _route(pol, ws, op, st[2], mode, (k, st[1]))
        elif st[0] == "evict":
            pol.evict_cache(st[1]); op.evict_cache(st[1])
        elif st[0] == "clear":
            pol.token_tree().clear(); op.token_tree().clear()
        elif st[0] == "urls":
            ws += [BasicWorker(u) for u in st[1][len(urls):]]
            urls = list(st[1])
            op.set_workers(urls)
            loads = list(loads) + [1] * (len(urls) - len(loads))
            _set_fleet(ws, op, loads)
        expect = fm.step(st, c0, op.token_tree().node_count())
        _same_state(pol, op, urls, (k, st[0]))
        scatters = _probe(pol, ws, op, mode, (k, "probe"))
        if expect is not None:
            assert scatters == (1 if expect == "scatter" else 0), (k, st[0], st[1], expect, scatters)
            seen[expect] += 1
    assert seen["scatter"] >= 4 and seen["full"] >= 3 and fm.inplace >= 1 and fm.growth >= 1
    hashes = op.hash_index("tokens")
    assert pol.hash_index_size("tokens") == len(hashes)
    for h, prefix in hashes.items():
        assert pol.hash_index_get(h, "tokens") == prefix
    _walk_many_device(pol, ws, op, [r for st in plan.steps if st[0] == "batch" for r in st[2]])


def _walk_many_device(pol, ws, op, reqs):
    """smgx_tree_walk_many_device over `reqs` in five batches: read-only, so together they equal one oracle snapshot call"""
    from smg_b200 import _lib
    L = _lib.load()
    model = pol._push_fleet(ws)
    entries = pol.token_tree().entries()
    ptrs = []

    def put(arr):
        err = _lib.new_err()
        p = L.smgx_device_alloc(pol._h.p, arr.nbytes + 16, C.byref(err))
        assert p, err.value
        ptrs.append(p)
        if arr.nbytes:
            pol._h.call("smgx_memcpy_h2d", C.c_void_p(p), arr.ctypes.data_as(C.c_void_p), arr.nbytes)
        return p

    nb = 5
    batches = [reqs[j::nb] for j in range(nb)]
    got_idx, got_info = [], []
    try:
        d_tok, d_off, d_out, d_info, ns = [], [], [], [], []
        for b in batches:
            off = np.zeros(len(b) + 1, np.uint32)
            np.cumsum([len(r) for r in b], out=off[1:])
            d_tok.append(put(P.cat(*b)))
            d_off.append(put(off))
            d_out.append(put(np.full(len(b), -7, np.int32)))
            d_info.append(put(np.zeros(len(b) * C.sizeof(_lib.DecisionInfo), np.uint8)))
            ns.append(len(b))
        arr = lambda xs: (C.c_void_p * len(xs))(*xs)
        pol._h.call("smgx_tree_walk_many_device", model, nb, arr(d_tok), arr(d_off), (C.c_uint32 * nb)(*ns), arr(d_out), arr(d_info))
        pol._h.call("smgx_synchronize")
        for j in range(nb):
            out = np.zeros(ns[j], np.int32)
            pol._h.call("smgx_memcpy_d2h", out.ctypes.data_as(C.c_void_p), C.c_void_p(d_out[j]), out.nbytes)
            got_idx += list(out)
            info = (_lib.DecisionInfo * ns[j])()
            pol._h.call("smgx_memcpy_d2h", C.cast(info, C.c_void_p), C.c_void_p(d_info[j]), C.sizeof(info))
            got_info += list(info)
    finally:
        for p in ptrs:
            L.smgx_device_free(pol._h.p, p)
    assert pol.token_tree().entries() == entries
    allq = [q for b in batches for q in b]
    off = np.zeros(len(allq) + 1, np.uint64)
    np.cumsum([len(q) for q in allq], out=off[1:])
    want, br, ma, _ = op.select_batch_tokens(P.cat(*allq), off, snapshot=True)
    for i, q in enumerate(allq):
        assert (want[i], br[i], ma[i], len(q)) == (got_idx[i], got_info[i].branch, got_info[i].matched, got_info[i].input), i
