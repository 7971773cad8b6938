"""Oracle request streams with the router's WorkerLoadGuard (routers/http/router.rs:319-321, worker/worker.rs:1067-1070): select_worker is
called one request at a time and the returned worker's load() is bumped before the next request.  The bumps live in a copy; the oracle's
fleet state is restored afterwards, so a call starts from its snapshot as the library's calls do."""
import numpy as np

from oracle import orc

BR = {name: i for i, name in enumerate(orc.BRANCHES)}


def stream(op, loads, texts=None, requests=None):
    """texts (request_text, string tree) or requests (token lists).  → (idx int32, branch uint8, matched, input, loads after the batch)."""
    reqs = texts if texts is not None else requests
    run = np.asarray(loads, np.uint64).copy()
    n = len(reqs)
    idx = np.full(n, -1, np.int32)
    br, ma, inp = np.zeros(n, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    for i, r in enumerate(reqs):
        op.set_state(loads=run)
        d = op.select_worker(request_text=r) if texts is not None else op.select_worker(tokens=r)
        br[i], ma[i], inp[i] = BR[d.branch], d.matched, d.input
        if d.idx is not None:
            idx[i] = d.idx
            run[d.idx] += 1
    op.set_state(loads=np.asarray(loads, np.uint64))
    return idx, br, ma, inp, run


def prefix_stream(oph, urls, loads, healthy, ring, requests):
    """prefix_hash: select_worker_impl one request at a time (None in `requests` = info.tokens None) with the pick's load bumped after each.
    → (idx int32, branch uint8, loads after the batch)."""
    run = np.asarray(loads, np.uint64).copy()
    idx, br = np.full(len(requests), -1, np.int32), np.zeros(len(requests), np.uint8)
    for i, r in enumerate(requests):
        w, name = oph.select_worker(urls, run, healthy, ring, r)
        br[i] = orc.PREFIX_BRANCHES.index(name)
        if w is not None:
            idx[i] = w
            run[w] += 1
    return idx, br, run


P2C_GOLDEN = 0x9E3779B97F4A7C15


def p2c_stream(op2, urls, loads, healthy, circuit, n, seed):
    """power_of_two: request i of a batch uses draws 2i and 2i + 1 of `seed`'s stream (draw k = finalise(seed + GOLDEN·k), k from 1), which
    are draws 1 and 2 of the stream seed + 2i·GOLDEN: so request i is select_worker alone on that seed, against the running loads."""
    run = np.asarray(loads, np.uint64).copy()
    idx, pairs, metric = np.full(n, -1, np.int32), np.full((n, 2), -1, np.int32), np.zeros(n, np.uint8)
    for i in range(n):
        w, pr, me, _ = op2.select_batch(urls, run, healthy, circuit, 1, (seed + 2 * i * P2C_GOLDEN) % 2**64)
        idx[i], pairs[i], metric[i] = w[0], pr[0], me[0]
        if w[0] >= 0:
            run[w[0]] += 1
    return idx, pairs, metric, run
