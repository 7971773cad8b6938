"""When event_slow_kernel runs behind event_lane_kernel / event_warp_kernel.

The lane and warp kernels queue a request for the slow kernel only when it has more than 32 blocks, more than one jump (blocks − 1 >
jump), or meets a Multi entry (a (position, content) key stored under two prefixes).  The host knows before the launch whether any of
these can happen: the launch's max_blocks, the index's jump and its count of Multi slots.  When none can, only the lane or warp kernel
is launched.  Each test compares every pick, branch and matched length with the oracle and counts the kernels of one call, in launches
of both kernels (the lane kernel from 256 requests per SM up, the warp kernel below)."""
import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth
from tests.test_gpu_event_sequences import (BS, MAX_BLOCKS, apply_ops, check, gpu_policy, oracle_policy, ragged, select_many, select_one,
                                            selected, set_fleet)

pytestmark = pytest.mark.gpu

W = 8
P = 32
BIG = 256 * 160   # the lane kernel on any GPU of up to 160 SMs


class Index:
    """The same stores on the GPU policy's indexer and on the oracle's; no Multi entry until xd is stored."""

    def __init__(self, jump, seed=11):
        urls = synth.worker_urls(W)
        self.pol, self.ws, self.ix = gpu_policy(urls, jump)
        self.op, self.oix = oracle_policy(urls, jump)
        self.rng = np.random.default_rng(seed)
        self.sid = 1
        self.a, self.b, self.md, self.xd, self.long = synth.gen_sequences(5, MAX_BLOCKS * BS, seed)
        self.xd[BS:2 * BS] = self.md[BS:2 * BS]   # block 1 of md under xd's prefix: a Multi entry at position 1 once both are stored
        self.store(0, self.a, P); self.store(1, self.a, 1); self.store(2, self.a, 20)   # a[:k], k ≥ 2: the count test fails
        self.store(3, self.b, P)
        self.store(4, self.long, MAX_BLOCKS)
        self.md_blocks = self.store(5, self.md, 8)
        fleet = (np.array([5, 3, 3, 9, 1, 0, 7, 2], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
        self.model = set_fleet(self.pol, self.ws, fleet)
        self.op.set_state(*fleet)

    def store(self, w, seq, depth):
        hs = orc.compute_request_content_hashes(seq[:depth * BS], BS)
        blocks = [(self.sid + i, int(h)) for i, h in enumerate(hs)]
        self.sid += depth
        apply_ops(self.ix, [("stored", w, blocks)]); apply_ops(self.oix, [("stored", w, blocks)])
        return [s for s, _ in blocks]

    def remove(self, w, seqs):
        apply_ops(self.ix, [("removed", w, seqs)]); apply_ops(self.oix, [("removed", w, seqs)])

    def noise(self, n):
        return self.rng.integers(0, synth.VOCAB, size=n, dtype=np.uint32)

    def shapes(self, max_blocks):
        """Full hits, failed count tests, drains that end in a miss, novel requests, the md / xd prefixes; up to max_blocks blocks."""
        a, b, md = self.a, self.b, self.md
        reqs = [a[:k * BS].copy() for k in range(1, P + 1)] + [b[:k * BS].copy() for k in range(1, P + 1)]
        reqs += [np.concatenate([b[:k * BS], self.noise((P - k) * BS)]) for k in (1, 5, 31)]
        reqs += [self.noise(BS), self.noise(P * BS), self.noise(BS - 1)]
        reqs += [md[:2 * BS].copy(), md[:8 * BS].copy(), self.xd[:2 * BS].copy(), self.xd[:8 * BS].copy()]
        reqs += [self.long[:n * BS].copy() for n in (33, 40, MAX_BLOCKS) if n <= max_blocks]
        return reqs

    def kernels_per_call(self, tag, reqs, cap, big):
        """Checks one call against the oracle (after a first call that flushes the index) and → the kernels the second call launched."""
        if big:
            reqs = [r.copy() for _ in range(-(-BIG // len(reqs))) for r in reqs]
        tokens, offsets, _ = ragged(reqs)
        oidx, obr, oma, _ = self.op.select_batch_tokens(tokens, offsets.astype(np.uint64))
        want = (np.asarray(oidx), np.asarray(obr), np.asarray(oma))
        select_one(self.pol, self.model, 0, reqs, cap)
        before = self.pol.kernel_launches()
        idx, info, lens = select_one(self.pol, self.model, 0, reqs, cap)
        n = self.pol.kernel_launches() - before
        check(tag, idx, info, lens, want)
        return n


@pytest.fixture(autouse=True)
def lane_kernel_selected():
    with selected("simple"):
        yield


@pytest.mark.parametrize("big", [False, True], ids=["warp_kernel", "lane_kernel"])
def test_slow_kernel_runs_only_while_the_index_holds_a_multi_entry(big):
    """Jump 64, at most 32 blocks: one kernel; a second prefix under one (position, content) makes a Multi entry: two; removing that
    prefix leaves the entry Multi (an entry never goes back to Single): two; removing the other one frees the slot: one again."""
    ix = Index(64)
    cap = P * BS
    assert ix.kernels_per_call("no Multi entry", ix.shapes(P), cap, big) == 1
    xd_blocks = ix.store(6, ix.xd, 2)
    assert ix.kernels_per_call("Multi entry at position 1", ix.shapes(P), cap, big) == 2
    ix.remove(6, xd_blocks)
    assert ix.kernels_per_call("one prefix left under the Multi entry", ix.shapes(P), cap, big) == 2
    ix.remove(5, ix.md_blocks)
    assert ix.kernels_per_call("Multi entry removed", ix.shapes(P), cap, big) == 1


@pytest.mark.parametrize("big", [False, True], ids=["warp_kernel", "lane_kernel"])
@pytest.mark.parametrize("jump, max_blocks", [(64, 33), (64, MAX_BLOCKS), (8, P), (30, P)])
def test_slow_kernel_runs_when_a_request_can_be_long_or_jump_twice(big, jump, max_blocks):
    """No Multi entry, but the launch allows more than 32 blocks, or more than one jump (max_blocks − 1 > jump): two kernels."""
    ix = Index(jump)
    assert ix.kernels_per_call(f"jump {jump}, max_blocks {max_blocks}", ix.shapes(max_blocks), max_blocks * BS, big) == 2


def test_one_kernel_at_the_largest_single_jump():
    """max_blocks − 1 = jump: every request is one jump, so the slow kernel is not launched."""
    ix = Index(31)
    assert ix.kernels_per_call("jump 31, 32 blocks", ix.shapes(P), P * BS, True) == 1


def test_multi_batch_launches_without_the_slow_kernel():
    """smgx_select_many_tokens_device with ragged batches (lane and warp kernel launches) on an index without a Multi entry."""
    ix = Index(64)
    shapes = ix.shapes(P)
    pick = lambda n: [shapes[i].copy() for i in ix.rng.integers(0, len(shapes), size=n)]   # noqa: E731
    for tag, sizes in (("warp kernel", (100, 300, 0, 57)), ("lane kernel", (20100, 15300, 0, 5057, 513))):
        batches = [pick(n) for n in sizes]
        select_many(ix.pol, ix.model, batches, P * BS)
        before = ix.pol.kernel_launches()
        got = select_many(ix.pol, ix.model, batches, P * BS)
        assert ix.pol.kernel_launches() - before == 1, tag
        for j, reqs in enumerate(batches):
            if reqs:
                tokens, offsets, _ = ragged(reqs)
                oidx = np.asarray(ix.op.select_batch_tokens(tokens, offsets.astype(np.uint64))[0])
                check(f"{tag}, batch {j}", got[j], None, None, (oidx, None, None))


@pytest.mark.parametrize("big", [False, True], ids=["warp_kernel", "lane_kernel"])
def test_multi_count_survives_a_rebuild_and_worker_clears(big):
    """The Multi slot count through a table rebuild (the index grows past half its capacity while a Multi entry is live), apply_cleared of
    one of its two workers (the entry stays Multi) and remove_worker of the other (the slot is freed)."""
    ix = Index(64)
    cap = P * BS
    ix.store(6, ix.xd, 2)
    assert ix.kernels_per_call("Multi entry", ix.shapes(P), cap, big) == 2
    ix.store(7, ix.noise(1500 * BS), 1500)   # 1024 slots at first: this rebuilds the table, more than once
    assert ix.kernels_per_call("after the rebuild", ix.shapes(P), cap, big) == 2
    ix.ix.apply_cleared(6); ix.oix.apply_cleared(6)
    assert ix.kernels_per_call("worker 6 cleared", ix.shapes(P), cap, big) == 2
    ix.ix.remove_worker(5); ix.oix.remove_worker(5)
    assert ix.kernels_per_call("worker 5 removed", ix.shapes(P), cap, big) == 1
