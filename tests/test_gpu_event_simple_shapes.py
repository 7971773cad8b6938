"""Request shapes at the edges of the default one-warp-per-request pick (block size 16, jump 64, ≤ 64 workers): one and two blocks (the
first and last probed positions coincide or are adjacent), a failed count test at every request length, and Multi entries at the last
position and in the middle of a drain.  The kernel hashes only the blocks it probes first and the rest only when the count test fails, so
each of these shapes takes a different route through it.  Every pick, branch and matched length is compared with the oracle, and the
picks whose answer follows from the stored sequences alone are checked against that answer too."""
import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth

pytestmark = pytest.mark.gpu

BS, JUMP, T = 16, 64, 512
P = T // BS


def test_short_requests_drains_and_multi_entries_match_the_oracle():
    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
    from smg_b200 import _lib
    _lib.load().smgx_set_event_path(1, 0)   # the default one-warp-per-request kernel
    cfg = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=BS)
    urls = synth.worker_urls(4)
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **cfg))
    ws = [BasicWorker(u) for u in urls]
    pol.init_workers(ws)
    mon = pol.kv_event_monitor(BS)
    ix = mon.create_indexer("unknown", JUMP)
    pol.set_kv_event_monitor(mon)
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **cfg)
    op.set_workers(urls)
    oix = orc.PositionalIndexer(JUMP)
    op.attach_indexer("unknown", oix)
    op.set_block_size("unknown", BS)
    op.set_kv_event_monitor(True)
    for u in urls:
        assert ix.intern_worker(u) == oix.intern_worker(u)

    a, mb, xb, mc, xc, noise = synth.gen_sequences(6, T, 7)
    xb[5 * BS:6 * BS] = mb[5 * BS:6 * BS]       # (5, block 5 of mb) is stored under two prefixes: a Multi entry
    xc[31 * BS:32 * BS] = mc[31 * BS:32 * BS]   # (31, block 31 of mc) likewise, at the last position of a 32-block request
    seq_id = [1]

    def store(w, seq, depth):
        hs = orc.compute_request_content_hashes(seq, BS)
        blocks = [(seq_id[0] + i, int(hs[i])) for i in range(depth)]
        seq_id[0] += depth
        ix.apply_stored(w, blocks)
        oix.apply_stored(w, blocks)

    store(0, a, P); store(1, a, 10)
    store(0, mb, P); store(1, mb, 20); store(2, xb, 8)
    store(0, mc, P); store(3, xc, P)
    loads = np.array([2, 1, 0, 0], np.uint64)   # between workers 0 and 1 a tie on the overlap goes to worker 1
    for w, l in zip(ws, loads):
        w.set_load(int(l))
    op.set_state(loads, [1] * 4, [1] * 4)

    reqs, known = [], []   # known: (request index, worker, matched blocks)
    for k in range(1, P + 1):
        reqs.append(a[:k * BS]); known.append((len(reqs) - 1, 1 if k <= 10 else 0, k))               # full hit, or a drain at 10
        if k < P:
            tail = np.concatenate([a[:k * BS], noise[k * BS:]])                                      # missing from k on
            reqs.append(tail); known.append((len(reqs) - 1, 1 if k <= 10 else 0, k))
    reqs.append(a[:BS + 7]); known.append((len(reqs) - 1, 1, 1))                                     # one block and a partial one
    reqs.append(a[:BS - 1])                                                                          # no full block
    reqs.append(noise)                                                                               # novel
    reqs.append(mb); known.append((len(reqs) - 1, 0, P))                                             # Multi at 5 inside the drain
    reqs.append(np.concatenate([mb[:3 * BS], noise[3 * BS:]])); known.append((len(reqs) - 1, 1, 3))  # the drain stops before the Multi
    reqs.append(np.concatenate([mb[:8 * BS], noise[8 * BS:]])); known.append((len(reqs) - 1, 1, 8))  # and after it
    reqs.append(xb[:8 * BS]); known.append((len(reqs) - 1, 2, 8))                                    # full hit past a Multi
    reqs.append(np.concatenate([xb[:8 * BS], noise[8 * BS:]])); known.append((len(reqs) - 1, 2, 8))  # drain through the Multi
    reqs.append(mc); known.append((len(reqs) - 1, 0, P))                                             # Multi at the last position
    reqs.append(xc); known.append((len(reqs) - 1, 3, P))
    reqs.append(mc[:31 * BS]); known.append((len(reqs) - 1, 0, 31))

    idx, info = pol.select_worker_batch(ws, reqs)
    lens = [len(r) for r in reqs]
    flat = np.concatenate(reqs).astype(np.uint32)
    offs = np.zeros(len(reqs) + 1, np.uint64); np.cumsum(lens, out=offs[1:])
    oidx, obr, oma, _ = op.select_batch_tokens(flat, offs)
    assert np.array_equal(idx, oidx)
    assert [i.branch for i in info] == list(obr)
    assert [i.matched * BS for i in info] == list(oma)
    for r, w, m in known:
        assert (idx[r], info[r].branch, info[r].matched) == (w, 2, m), f"request {r} ({lens[r]} tokens)"
