"""event_lane_kernel's drains through the run arena, against the oracle.

Every apply_stored call writes its blocks into one run of consecutive records (record index = anchor + position), and phase B reads a
drained position's record beside its tokens, starting from the anchor of the position-0 entry; a live record of the key is the entry,
and anything else (a dead record, another run's record, no record) falls back to the tag walk and the slot, which re-anchors the drain
at the run that holds the key.  Each test builds index histories that put the records a drain meets in each of those states — runs
broken up by other workers' and chained stores, records killed, rewritten, compacted away and moved — repeated into launches of more
than BIG requests so that the lane kernel runs, and compares every pick, branch and matched length with the oracle."""
import numpy as np
import pytest

from tests.test_gpu_event_lane import BIG, P, Index
from tests.test_gpu_event_sequences import BS, apply_ops, selected
from smg_b200 import synth
from oracle import orc

pytestmark = pytest.mark.gpu


class RunIndex(Index):
    """test_gpu_event_lane's index plus sequences stored so that their runs are whole, chained, broken up and rewritten."""

    def __init__(self):
        super().__init__(64)
        seqs = iter(synth.gen_sequences(48, P * BS, 2029))   # a seed whose blocks the base index does not share
        # c[k]: 32 blocks on worker 0 (one whole run), the first k on worker 1 (a run of dead records, the live ones' payload rewritten)
        self.c = {k: next(seqs) for k in range(1, 32)}
        for k, s in self.c.items():
            self.store(0, s, P); self.store(1, s, k)
        # chained: 32 blocks stored over 2, 3 and 4 calls, each continuing from the last block of the one before
        self.chained = {}
        for cuts in ((11,), (5, 20), (1, 9, 17)):
            s = next(seqs)
            self.store_chain(3, s, cuts)
            self.chained[cuts] = s
        # shared: worker 4 stores the first 5 blocks, worker 5 then all 32 (its run: positions 0..4 dead, 5..31 live)
        self.shared = next(seqs)
        self.store(4, self.shared, 5); self.store(5, self.shared, P)
        # hole: 32 blocks on worker 0, block 12 removed (its record dead), then stored again by a one-block chained call
        self.hole = next(seqs)
        ids = self.store(0, self.hole, P)
        self.remove(0, [ids[12]])
        self.hole_ids = ids
        # mm: a Multi entry at position 12, inside worker 0's run (Single → Multi rewrites the record)
        self.mm, xm = next(seqs), next(seqs)
        xm[12 * BS:13 * BS] = self.mm[12 * BS:13 * BS]
        self.store(0, self.mm, 20); self.store(1, self.mm, 14); self.store(2, xm, 13)
        # twice: worker 6 stores a sequence worker 7 then stores as well (bits added to live records), later removed again
        self.twice = next(seqs)
        self.store(6, self.twice, P)
        self.twice_ids = self.store(7, self.twice, P)

    def store_chain(self, w, seq, cuts):
        """seq's 32 blocks in len(cuts) + 1 apply_stored calls, each with the previous call's last block as parent."""
        hs = orc.compute_request_content_hashes(seq[:P * BS], BS)
        ids = list(range(self.sid, self.sid + P))
        self.sid += P
        bounds = (0,) + tuple(cuts) + (P,)
        for lo, hi in zip(bounds, bounds[1:]):
            blocks = [(ids[i], int(hs[i])) for i in range(lo, hi)]
            parent = ids[lo - 1] if lo else None
            self.ix.apply_stored(w, blocks, parent); self.oix.apply_stored(w, blocks, parent)
        return ids

    def store_again(self, w, seq, pos, ids):
        """Block `pos` of seq alone, chained to block pos - 1 (a run of one record)."""
        h = int(orc.compute_request_content_hashes(seq[:(pos + 1) * BS], BS)[pos])
        blocks = [(ids[pos], h)]
        self.ix.apply_stored(w, blocks, ids[pos - 1]); self.oix.apply_stored(w, blocks, ids[pos - 1])

    def remove(self, w, ids):
        apply_ops(self.ix, [("removed", w, ids)]); apply_ops(self.oix, [("removed", w, ids)])

    def each(self, method, *args):
        getattr(self.ix, method)(*args); getattr(self.oix, method)(*args)

    def partial_hits(self):
        """For every k in 1..31: k stored blocks then novel ones, the whole stored sequence (narrows at k) and a request one block past k."""
        reqs = []
        for k, s in self.c.items():
            reqs += [self.tail(s, k), s[:P * BS].copy(), s[:min(k + 1, P) * BS].copy()]
        return reqs

    def run_shapes(self):
        reqs = []
        for s in list(self.chained.values()) + [self.shared, self.hole, self.twice]:
            reqs += [s[:n * BS].copy() for n in (2, 5, 6, 9, 12, 13, 18, 21, 32)]
            reqs += [self.tail(s, k) for k in (1, 5, 6, 11, 12, 13, 17, 20, 31)]
        reqs += [self.mm[:n * BS].copy() for n in (12, 13, 14, 20)] + [self.tail(self.mm, 14, 20)]
        return reqs

    def mix(self, reqs):
        """reqs among full hits and novel requests, in the bench's proportions around them."""
        out = []
        for r in reqs:
            out += [r, self.b[:P * BS].copy(), self.a[:P * BS].copy(), self.noise(P * BS)]
        return out


@pytest.fixture(scope="module")
def runs():
    with selected("simple"):
        yield RunIndex()


@pytest.mark.parametrize("shift", [0, 1, 3])
def test_partial_hits_of_every_length(runs, shift):
    reqs = ([runs.noise(shift)] if shift else []) + runs.mix(runs.partial_hits())
    _, info = runs.check_one(f"partial hits, shift {shift}", reqs)
    assert (info["branch"] == 2).sum() > 1000


@pytest.mark.parametrize("shift", [0, 1, 3])
def test_chained_shared_and_rewritten_runs(runs, shift):
    """Runs split over chained calls, a prefix whose position 0 lives in another worker's shorter run, a removed middle block, a
    Multi entry inside a run (event_slow_kernel), a sequence a second worker stored as well."""
    reqs = ([runs.noise(shift)] if shift else []) + runs.mix(runs.run_shapes())
    runs.check_one(f"runs, shift {shift}", reqs)


def test_index_changes_between_picks():
    """The same requests after each change: a removed block stored again, a second worker's copy removed, a worker cleared, a
    worker removed."""
    with selected("simple"):
        ix = RunIndex()
        reqs = ix.mix(ix.partial_hits() + ix.run_shapes())
        ix.check_one("before", reqs)
        ix.store_again(0, ix.hole, 12, ix.hole_ids)
        ix.check_one("hole stored again", reqs)
        ix.remove(7, ix.twice_ids)
        ix.check_one("second copy removed", reqs)
        ix.each("apply_cleared", 1)
        ix.check_one("worker 1 cleared", reqs)
        ix.each("remove_worker", 0)
        ix.check_one("worker 0 removed", reqs)


def test_growth_and_compaction_between_picks():
    """Two rounds of thousands of short sequences stored and then removed, with picks in between: the slot table grows and is rebuilt,
    and the arena is compacted (at the rebuilds, and by a store once dead records outnumber the live entries), which moves the runs
    that are kept and drops the dead ones."""
    with selected("simple"):
        ix = RunIndex()
        reqs = ix.mix(ix.partial_hits() + ix.run_shapes())
        ix.check_one("before", reqs)
        for rnd in range(2):
            filler = synth.gen_sequences(3000, 8 * BS, 4099 + rnd)
            ids = [ix.store(2 + i % 6, s, 8) for i, s in enumerate(filler)]
            ix.check_one(f"round {rnd}, stored", reqs + ix.mix([f[:8 * BS].copy() for f in filler[:64]]))
            for i, sid in enumerate(ids):
                ix.remove(2 + i % 6, sid)
            ix.store_again(0, ix.hole, 12, ix.hole_ids)
            ix.check_one(f"round {rnd}, removed, hole stored again", reqs)
            ix.remove(0, [ix.hole_ids[12]])
            ix.check_one(f"round {rnd}, hole removed again", reqs)
