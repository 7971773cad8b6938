"""Request shapes at the edges of event_lane_kernel, the event-driven pick for plain picks (≤ 64 workers, block size 16) in launches of at
least 256 requests per SM; smaller launches run event_warp_kernel, one warp per request.

The kernel decides one request per thread (phase A: blocks 0 and last hashed, both probes, the count-only jump test) and drains the
requests whose count test failed across the CTA's warps, two per round (phase B); what needs the rolling prefix hash or more than one
jump goes to event_slow_kernel through a device queue, from phase A or from phase B.  Each test below builds request shapes that take
one of those routes, repeated into launches of more than BIG requests (the lane kernel on any GPU of up to 160 SMs) and, where noted, in
small launches (the warp kernel), with sizes that do and do not fill whole warps and CTAs, and compares every pick, branch and matched
length with the oracle."""
import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth
from tests.test_gpu_event_sequences import (BS, IMBALANCED, MAX_BLOCKS, NO_HEALTHY, Device, apply_ops, build_plan, check, gpu_policy,
                                            launch_one, oracle_policy, ragged, run_oracle, select_many, select_one, selected, set_fleet)

pytestmark = pytest.mark.gpu

W = 8
P = 32
BIG = 256 * 160


class Index:
    """The same stores on the GPU policy's indexer and on the oracle's; the request shapes built from them."""

    def __init__(self, jump, seed=5):
        urls = synth.worker_urls(W)
        self.pol, self.ws, self.ix = gpu_policy(urls, jump)
        self.op, self.oix = oracle_policy(urls, jump)
        self.rng = np.random.default_rng(seed)
        self.sid = 1
        a, b, e, long_, md, xd, mb, xb, mc, xc = synth.gen_sequences(10, MAX_BLOCKS * BS, seed)
        xd[BS:2 * BS] = md[BS:2 * BS]              # (1, block 1 of md) under two prefixes: a Multi entry at position 1
        xb[4 * BS:5 * BS] = mb[4 * BS:5 * BS]      # (4, block 4 of mb): inside the drain of mb[:8]
        xc[5 * BS:6 * BS] = mc[5 * BS:6 * BS]      # (5, block 5 of mc): the last position of mc[:6]
        self.store(0, a, P); self.store(1, a, 1); self.store(2, a, 20)   # a[:k], k ≥ 2: the count test fails at every length
        self.store(3, b, P)                                                # b[:k]: full hits; with a novel tail: a drain to a miss
        self.store(4, long_, MAX_BLOCKS)
        self.store(0, md, 8); self.store(1, md, 1); self.store(2, xd, 2)
        self.store(0, mb, 8); self.store(1, mb, 6); self.store(2, xb, 5)
        self.store(0, mc, 6); self.store(3, xc, 6)
        gone = self.store(5, e, 4)                                         # stored, then removed: nothing (or an empty set) at position 0
        apply_ops(self.ix, [("removed", 5, gone)]); apply_ops(self.oix, [("removed", 5, gone)])
        self.a, self.b, self.e, self.long, self.md, self.mb, self.mc, self.xb, self.xc = a, b, e, long_, md, mb, mc, xb, xc
        self.balanced((np.array([5, 3, 3, 9, 1, 0, 7, 2], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8)))

    def store(self, w, seq, depth):
        hs = orc.compute_request_content_hashes(seq[:depth * BS], BS)
        blocks = [(self.sid + i, int(h)) for i, h in enumerate(hs)]
        self.sid += depth
        apply_ops(self.ix, [("stored", w, blocks)]); apply_ops(self.oix, [("stored", w, blocks)])
        return [s for s, _ in blocks]

    def balanced(self, fleet):
        self.model = set_fleet(self.pol, self.ws, fleet)
        self.op.set_state(*fleet)

    def noise(self, n):
        return self.rng.integers(0, synth.VOCAB, size=n, dtype=np.uint32)

    def tail(self, seq, k, n=P):   # the first k blocks of seq, then novel blocks up to n
        return np.concatenate([seq[:k * BS], self.noise((n - k) * BS)])

    def drains(self, n):   # n requests whose count test fails and whose drain needs no generic search
        return [self.a[:(2 + i % (P - 1)) * BS].copy() if i % 2 else self.tail(self.b, 1 + i % (P - 1)) for i in range(n)]

    def shapes(self):
        a, b = self.a, self.b
        reqs = [a[:BS].copy(), a[:2 * BS].copy(), b[:BS].copy(), b[:2 * BS].copy(), self.tail(b, 1, 2),   # one and two blocks
                self.noise(BS), self.noise(P * BS), self.noise(BS - 1), self.e[:4 * BS].copy()]          # novel, no full block, empty set
        reqs += [a[:k * BS].copy() for k in range(2, P + 1)]                                                # failed count test, 2..32 blocks
        reqs += [b[:k * BS].copy() for k in range(1, P + 1)]                                                # full hits
        reqs += [self.tail(b, k, n) for k, n in ((1, 9), (5, 32), (31, 32), (16, 17))]                     # drains that end in a miss
        reqs += [self.long[:n * BS].copy() for n in (33, 40, MAX_BLOCKS)]                                   # more than 32 blocks
        reqs += [self.md[:2 * BS].copy(), self.md[:8 * BS].copy(), self.tail(self.md, 1, 8)]                # Multi at 1: phase A, phase B
        reqs += [self.mb[:8 * BS].copy(), self.mb[:5 * BS].copy(), self.xb[:5 * BS].copy()]                 # Multi mid-drain, at last
        reqs += [self.mc[:6 * BS].copy(), self.xc[:6 * BS].copy(), self.mc[:5 * BS].copy()]                 # Multi at last, one short of it
        return reqs

    def want(self, reqs):
        tokens, offsets, _ = ragged(reqs)
        idx, br, ma, _ = self.op.select_batch_tokens(tokens, offsets.astype(np.uint64))
        return np.asarray(idx), np.asarray(br), np.asarray(ma)

    def check_one(self, tag, reqs, cap=0, big=True):
        if big and len(reqs) < BIG:   # repeated into a launch that takes the lane kernel
            reqs = [r.copy() for _ in range(-(-BIG // len(reqs))) for r in reqs]
        idx, info, lens = select_one(self.pol, self.model, 0, reqs, cap)
        check(tag, idx, info, lens, self.want(reqs))
        return idx, info

    def check_many(self, tag, batches):
        for j, got in enumerate(select_many(self.pol, self.model, batches, 0)):
            if len(batches[j]):
                check(f"{tag}, batch {j}", got, None, None, self.want(batches[j]))


@pytest.fixture(scope="module", params=[64, 8], ids=["jump64", "jump8"])
def index(request):
    with selected("simple"):
        yield Index(request.param)


@pytest.mark.parametrize("shift", [0, 1, 3])
def test_request_shapes_match_the_oracle(index, shift):
    """Every route through phase A and B, with token offsets 16 B aligned (shift 0) and not (a shift-token request in front)."""
    reqs = ([index.noise(shift)] if shift else []) + index.shapes()
    idx, info = index.check_one(f"shapes, shift {shift}", reqs)
    assert (info["branch"] == 2).sum() > 50


def test_drain_queues_fill_a_warp_and_outnumber_the_warps(index):
    """A warp whose 32 requests all drain; CTAs with 40, 256 and 13 drains (several rounds per warp, pairs and a lone last drain).  The
    list is 781 requests long and repeated into a launch of more than BIG requests."""
    full = index.drains(32) + [index.b[:P * BS].copy() for _ in range(224)]   # warp 0 of a CTA of 256 drains everything, the rest are hits
    reqs = full + index.drains(40) + [index.b[:3 * BS].copy() for _ in range(216)] + index.drains(256) + index.drains(13)
    index.check_one("drains", reqs)


@pytest.mark.parametrize("total", [1, 31, 33, 255, 257, BIG + 1, BIG + 31, BIG + 33, BIG + 255, BIG + 257])
def test_ragged_totals(index, total):
    """Totals that leave the last warp and CTA partly empty, in small launches (warp kernel) and large ones (lane kernel)."""
    shapes = index.shapes()
    order = index.rng.permutation(max(total, len(shapes)))[:total] % len(shapes)
    index.check_one(f"total {total}", [shapes[i].copy() for i in order], big=False)


def test_multi_batch_launches_straddle_batch_boundaries(index):
    """smgx_select_many_tokens_device: ragged batch sizes (batch found by its first global index) and equal ones (by division), both
    with CTAs that span two batches, and an empty batch in between."""
    shapes = index.shapes() + index.drains(40)
    pick = lambda n: [shapes[i].copy() for i in index.rng.integers(0, len(shapes), size=n)]   # noqa: E731
    index.check_many("ragged", [pick(n) for n in (100, 300, 0, 57, 256, 3)])
    index.check_many("uniform", [pick(200) for _ in range(3)])
    index.check_many("ragged, lane kernel", [pick(n) for n in (20100, 15300, 0, 5057, 513, 3)])
    index.check_many("uniform, lane kernel", [pick(13700) for _ in range(3)])


@pytest.mark.parametrize("fleet", ["imbalanced", "no_healthy", "one_down"])
def test_fleet_states(index, fleet):
    loads, healthy, circuit = np.array([5, 3, 3, 9, 1, 0, 7, 2], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8)
    if fleet == "imbalanced":
        loads[2] = 500
    elif fleet == "no_healthy":
        healthy[:] = 0
    else:
        healthy[0] = 0; circuit[3] = 0
    index.balanced((loads, healthy, circuit))
    try:
        idx, info = index.check_one(fleet, index.shapes() + index.drains(20))
        if fleet == "imbalanced":
            assert set(info["branch"]) == {IMBALANCED}
        elif fleet == "no_healthy":
            assert set(info["branch"]) == {NO_HEALTHY} and set(idx) == {-1}
    finally:
        index.balanced((np.array([5, 3, 3, 9, 1, 0, 7, 2], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8)))


def test_request_over_the_cap(index):
    """A request longer than max_request_tokens: -1, branch 255, reported once by the next synchronise; the rest are answered."""
    from smg_b200 import SmgxError
    reqs = [r for r in index.shapes() if len(r) <= P * BS]
    reqs = [r.copy() for _ in range(-(-BIG // len(reqs))) for r in reqs]
    reqs.insert(7, index.long[:40 * BS].copy())
    dev = Device(index.pol)
    try:
        read = launch_one(index.pol, dev, index.model, 0, reqs, P * BS)
        with pytest.raises(SmgxError, match="exceeded max_tokens_per_request"):
            index.pol._h.call("smgx_synchronize")
        index.pol._h.call("smgx_synchronize")
        idx, info, lens = read()
    finally:
        dev.free()
    assert (idx[7], info["branch"][7]) == (-1, 255)
    keep = np.arange(len(reqs)) != 7
    oidx, obr, oma = index.want(reqs)
    check("over the cap", idx[keep], info[keep], lens[keep], (oidx[keep], obr[keep], oma[keep]))


@pytest.mark.parametrize("value", [0, 4, 5, 6])
def test_every_nonzero_selection_runs_the_lane_kernel(value):
    """smgx_set_event_simple: 4, 5 and 6 launch event_lane_kernel + event_slow_kernel (two kernels per call), 0 the fused kernel (one)."""
    from smg_b200 import _lib
    ix = Index(64)
    with selected("fused"):
        _lib.load().smgx_set_event_simple(value)
        reqs = ix.shapes()
        ix.check_one("first call (flushes the index and the fleet)", reqs)
        before = ix.pol.kernel_launches()
        ix.check_one(f"SMGX_EVENT_SIMPLE={value}", reqs)
        assert ix.pol.kernel_launches() - before == (2 if value else 1)


def test_launch_sequence_with_the_lane_kernel_selected_as_4():
    """The slow queue's count and exit counter across growing and shrinking launches (test_gpu_event_sequences' plan, jump 8; its
    launches are small, so this runs event_warp_kernel; the lane kernel's launches above share each policy's queue with small ones)."""
    from smg_b200 import _lib
    jump = 8
    plan, want = build_plan(jump), run_oracle(jump)
    with selected("simple"):
        _lib.load().smgx_set_event_simple(4)
        pol, ws, ix = gpu_policy(plan["urls"], jump)
        apply_ops(ix, plan["init"])
        for i, (st, exp) in enumerate(zip(plan["steps"], want)):
            apply_ops(ix, st["ops"])
            model = set_fleet(pol, ws, st["fleet"])
            tag = f"call {i} ({st['mix']}, lane {st['lane']}, n = {[len(b) for b in st['batches']]})"
            if st["many"]:
                for j, (got, e) in enumerate(zip(select_many(pol, model, st["batches"], st["cap"]), exp)):
                    check(f"{tag}, batch {j}", got, None, None, e)
            else:
                idx, info, lens = select_one(pol, model, st["lane"], st["batches"][0], st["cap"])
                check(tag, idx, info, lens, exp[0])
