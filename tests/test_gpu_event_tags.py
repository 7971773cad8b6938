"""The index's tag array (one byte per slot, derived on the device) under churn, against the oracle.

Lookups walk collision chains in the tags and read a slot only where the tag matches, so a tag array that falls behind the slots
(a flush path that forgets it, a tombstone that keeps a live tag, a rebuild that leaves old tags) shows up as a wrong pick, branch or
matched length.  Starting from the smallest table (1024 slots, filled to half before every growth, so chains cross tag sectors and wrap
at the end of the table), each step below changes the index, and every step is followed by requests that probe every stored key,
removed keys and absent keys: in launches large enough for event_lane_kernel, in small launches (event_warp_kernel), and requests of
more than 32 blocks (event_slow_kernel)."""
import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth
from tests.test_gpu_event_sequences import (BS, MAX_BLOCKS, apply_ops, check, gpu_policy, oracle_policy, ragged, select_one, selected,
                                            set_fleet)

pytestmark = pytest.mark.gpu

W = 8
P = 32
BIG = 256 * 160   # more requests than 256 per SM on any GPU of up to 160 SMs: the lane kernel


class Churn:
    def __init__(self, jump, seed):
        urls = synth.worker_urls(W)
        self.pol, self.ws, self.ix = gpu_policy(urls, jump)
        self.op, self.oix = oracle_policy(urls, jump)
        self.rng = np.random.default_rng(seed)
        self.seqs = synth.gen_sequences(160, MAX_BLOCKS * BS, seed)
        self.sid = 1
        self.stored = {}   # sequence → [(worker, seq ids)]
        fleet = (np.array([5, 3, 3, 9, 1, 0, 7, 2], np.uint64), np.ones(W, np.uint8), np.ones(W, np.uint8))
        self.model = set_fleet(self.pol, self.ws, fleet)
        self.op.set_state(*fleet)

    def both(self, fn, *args):
        getattr(self.ix, fn)(*args)
        getattr(self.oix, fn)(*args)

    def store(self, s, w, depth):
        hs = orc.compute_request_content_hashes(self.seqs[s][:depth * BS], BS)
        blocks = [(self.sid + i, int(h)) for i, h in enumerate(hs)]
        self.sid += depth
        apply_ops(self.ix, [("stored", w, blocks)]); apply_ops(self.oix, [("stored", w, blocks)])
        self.stored.setdefault(s, []).append((w, [b for b, _ in blocks]))

    def remove_tail(self, s, keep):   # removes blocks keep.. of every copy of sequence s: tombstones on the chains of later keys
        for w, ids in self.stored.get(s, []):
            apply_ops(self.ix, [("removed", w, ids[keep:])]); apply_ops(self.oix, [("removed", w, ids[keep:])])

    def requests(self):
        """Every sequence ever used, at full length and cut at every block count, plus its tail replaced by novel tokens and pure noise."""
        reqs = []
        for s in range(len(self.seqs)):
            seq = self.seqs[s]
            reqs += [seq[:k * BS].copy() for k in range(1, P + 1)]
            reqs.append(np.concatenate([seq[:5 * BS], self.rng.integers(0, synth.VOCAB, size=(P - 5) * BS, dtype=np.uint32)]))
        reqs += [self.seqs[s][:n * BS].copy() for s in range(0, len(self.seqs), 7) for n in (33, 48, MAX_BLOCKS)]   # the slow kernel
        reqs += [self.rng.integers(0, synth.VOCAB, size=n * BS, dtype=np.uint32) for n in (1, 2, 17, 32, 40)]
        return reqs

    def want(self, reqs):
        tokens, offsets, _ = ragged(reqs)
        return tuple(np.asarray(x) for x in self.op.select_batch_tokens(tokens, offsets.astype(np.uint64))[:3])

    def check_all(self, tag):
        reqs = self.requests()
        want = self.want(reqs)
        idx, info, lens = select_one(self.pol, self.model, 0, reqs, 0)                      # small launch: the warp kernel
        check(f"{tag}, {len(reqs)} requests", idx, info, lens, want)
        big = [r for _ in range(-(-BIG // len(reqs))) for r in reqs]
        idx, info, lens = select_one(self.pol, self.model, 0, big, 0)                       # large launch: the lane kernel
        check(f"{tag}, {len(big)} requests", idx, info, lens, self.want(big))
        return want


@pytest.mark.parametrize("jump", [64, 8])
def test_tags_follow_the_slots_under_churn(jump):
    with selected("simple"):
        c = Churn(jump, seed=11 + jump)
        for s in range(40):                        # 1280 entries: grows 1024 → 4096 slots (rebuild: the bulk upload)
            c.store(s, s % W, P)
        c.store(40, 1, 48)                         # more than 32 blocks
        want = c.check_all("after growth")
        assert (want[1] == 2).sum() > 1000         # overlaps found
        for s in range(0, 40, 4):                  # 10 tails of 16 blocks: far fewer dirty slots than 1/8 of the table (the scatter)
            c.remove_tail(s, 16)
        c.check_all("after removals")
        for s in range(0, 40, 4):                  # stored again on other workers: inserts that re-use tombstones
            c.store(s, (s + 3) % W, 24)
        c.check_all("after re-stores")
        c.both("apply_cleared", 2)
        c.check_all("after apply_cleared")
        c.both("remove_worker", 5)
        c.check_all("after remove_worker")
        for s in range(41, 160):                   # ≈ 3800 more entries: a second growth, then a dense table
            c.store(s, s % W, P)
        c.check_all("after the second growth")
        for s in range(41, 160):                   # ≈ 3700 tombstones in one flush: more than 1/8 of the slots dirty (the bulk upload)
            c.remove_tail(s, 1)
        c.check_all("after bulk removals")
        c.store(41, 4, 8)
        c.check_all("after one store")             # a handful of dirty slots (the scatter) behind a bulk upload
