"""The drains of event_lane_kernel's phase B against the oracle, at the edges of their segments.

Phase B drains a failed count test in segments of 8 positions (1..8, 9..16, 17..24, 25..31), four drains per warp, and stops a drain
where the reference's linear scan stops: at the first missing position, when the active set is empty, or at an entry that needs the
generic search.  A finished drain's slot takes the next queued drain of the CTA.  Each test builds request shapes around those edges,
repeated into launches of more than BIG requests so that the lane kernel runs, and compares every pick, branch and matched length with
the oracle."""
import numpy as np
import pytest

from tests.test_gpu_event_lane import BIG, P, Index
from tests.test_gpu_event_sequences import BS, apply_ops, selected
from smg_b200 import synth

pytestmark = pytest.mark.gpu

EDGES = (3, 8, 9, 13, 16, 17, 20, 24, 25, 30, 31)   # inside the first and third segments, and on both sides of every boundary


class SegIndex(Index):
    """test_gpu_event_lane's index plus sequences whose drains end, narrow or bail at chosen positions."""

    def __init__(self):
        super().__init__(64)
        seqs = synth.gen_sequences(31 + len(EDGES) + 3, P * BS, 1009)   # another seed than the base index's, which shares no block
        # c[k]: 32 blocks on worker 0, the first k on worker 1 — a 32-block request drops to {0} at k, a k-block prefix plus novel
        # blocks ends at k
        self.c = {k: seqs[k - 1] for k in range(1, 32)}
        for k, s in self.c.items():
            self.store(0, s, P); self.store(1, s, k)
        # x[m]: 32 blocks on workers 0 and 1, the first m on worker 2.  With block m replaced the request misses at m, and positions
        # m+1.. are present again with the smaller set {0, 1}: the scan must end at m
        self.x = {m: seqs[31 + i] for i, m in enumerate(EDGES)}
        for m, s in self.x.items():
            self.store(0, s, P); self.store(1, s, P); self.store(2, s, m)
        # y: 32 blocks on workers 0 and 1, 28 on worker 2, worker 1's block 12 removed: {0, 2} at 12, then {0, 1, 2} and {0, 1} —
        # counts at or above the narrowed set's, which the retain guard keeps from changing it
        self.y = seqs[31 + len(EDGES)]
        self.store(0, self.y, P); self.store(2, self.y, 28)
        ids = self.store(1, self.y, P)
        apply_ops(self.ix, [("removed", 1, [ids[12]])]); apply_ops(self.oix, [("removed", 1, [ids[12]])])
        # mm: a Multi entry at position 12 (second segment): block 12 of mm also stored under another prefix (xm)
        self.mm, xm = seqs[32 + len(EDGES)], seqs[33 + len(EDGES)].copy()
        xm[12 * BS:13 * BS] = self.mm[12 * BS:13 * BS]
        self.store(0, self.mm, 20); self.store(1, self.mm, 14); self.store(2, xm, 13)
        self.edges = self.edge_shapes()

    def edge_shapes(self):
        reqs = [self.c[k][:n * BS].copy() for k in self.c for n in range(2, P + 1) if n > k or n in (2, 8, 9, 17, 25, 32)]
        reqs += [self.tail(self.c[k], k) for k in self.c]                                   # stored prefix ends at k
        reqs += [self.tail(self.c[k], k, n) for k in (1, 7, 8, 15, 16, 24) for n in (k + 1, k + 2)]
        for m, s in self.x.items():
            r = s[:P * BS].copy()
            r[m * BS:(m + 1) * BS] = self.noise(BS)
            reqs += [r, r[:(m + 2) * BS].copy(), s[:P * BS].copy()]
        reqs += [self.y[:n * BS].copy() for n in (13, 14, 29, 30, P)]
        reqs += [self.mm[:n * BS].copy() for n in (12, 13, 14, 20)]                           # Multi before, at and inside the drain
        return reqs

    def cta(self, n_drains):
        """256 requests of which n_drains fail their count test (spread over the CTA) and the rest are full hits."""
        drains = self.edges
        pick = self.rng.integers(0, len(drains), size=n_drains)
        where = set(self.rng.choice(256, size=n_drains, replace=False).tolist())
        it = iter(pick)
        return [drains[next(it)].copy() if i in where else self.b[:P * BS].copy() for i in range(256)]


@pytest.fixture(scope="module")
def seg():
    with selected("simple"):
        yield SegIndex()


def test_edge_shapes_match_the_oracle(seg):
    _, info = seg.check_one("segment edges", seg.edges)
    assert (info["branch"] == 2).sum() > 1000


@pytest.mark.parametrize("shift", [0, 1, 3])
def test_cta_queues_of_every_length(seg, shift):
    """CTAs holding 0, 1, 3, 4, 5, 31, 32, 33 and 256 drains: fewer, as many and more than the 32 drain slots of a CTA, so that slots
    stay idle, take one drain each, or are refilled.  shift tokens on the first request move every later token range off 16 B."""
    ctas = []
    while len(ctas) * 256 < BIG:
        for n in (0, 1, 3, 4, 5, 31, 32, 33, 256):
            ctas += [seg.cta(n)]
    reqs = [r for c in ctas for r in c]
    reqs[0] = np.concatenate([reqs[0], seg.noise(shift)]) if shift else reqs[0]
    seg.check_one(f"CTA queues, shift {shift}", reqs)


def test_cta_straddles_two_batches(seg):
    """A CTA whose requests, drains among them, come from two batches of one launch; equal and unequal batch sizes."""
    half = 256 * 83 + 128                                          # batch 1 starts inside CTA 83, which holds 256 drains
    reqs = [r for _ in range(-(-2 * half // 768)) for n in (33, 5, 256) for r in seg.cta(n)]
    assert 2 * half >= BIG
    cut = 256 * 32 + 100                                           # inside CTA 32, which holds 256 drains
    seg.check_many("straddle, ragged", [reqs[:cut], reqs[cut:]])
    seg.check_many("straddle, uniform", [reqs[:half], reqs[half:2 * half]])
