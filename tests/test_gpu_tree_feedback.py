"""Load feedback in the token-tree and string-tree modes (smgx_set_load_feedback_policies with SMGX_FEEDBACK_CACHE_AWARE): a batch is the
request stream of a router that takes a WorkerLoadGuard after every pick (routers/http/router.rs:319-321).  Oracle = select_worker called
one request at a time with the picked worker's load bumped after each pick (tests/feedback_stream.py).  Picks, branches, matched / input
counts, the final trees with their timestamps, hash_index, processed counts and the loads after the batch must all agree."""
import json
import os
import random

import numpy as np
import pytest

from oracle import orc
from smg_b200 import synth
from tests import feedback_stream as FS

pytestmark = pytest.mark.gpu

CFG = dict(cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=16)
GONE = "http://gone-worker:1"          # a tenant whose URL is not in the worker slice
GOLD = os.path.join(os.path.dirname(__file__), "golden")
T, B = 96, 1024


def _pair(n_workers, feedback=True, empty_indexer=False, tokenizer=False):
    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
    urls = synth.worker_urls(n_workers)
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **CFG), max_batch=8192)
    ws = [BasicWorker(u) for u in urls]
    pol.init_workers(ws)
    orc.reset_globals()
    op = orc.CacheAwarePolicy(eviction_interval_secs=0, **CFG)
    op.set_workers(urls)
    if empty_indexer:      # an event-mode model whose indexer holds nothing yet routes through the token tree
        mon = pol.kv_event_monitor(16)
        mon.create_indexer("unknown", 64)
        pol.set_kv_event_monitor(mon)
        op.attach_indexer("unknown", orc.PositionalIndexer(64))
        op.set_kv_event_monitor(True)
    if tokenizer:
        g = json.load(open(os.path.join(GOLD, "bpe_vectors.json")))
        pol.load_tiktoken_tokenizer(os.path.join(GOLD, "synth_vocab.tiktoken"), g["specials"])
    if feedback:
        pol.set_load_feedback_all_modes(True)
    return pol, ws, op


def _fleets(n, seed):
    """(name, loads, healthy) per batch: Poisson loads; a gate open at the start that closes inside the batch; an unhealthy worker pinning
    the minimum; loads above 2^24 (f32 conversions round)."""
    rng = np.random.default_rng(seed)
    ones = np.ones(n, np.uint8)
    gate = np.full(n, 80, np.uint64)
    gate[:4] = 0           # max - min = 80 > 64: min-load picks fill the four until they reach 16 (64 picks), then the gate closes
    pin = synth.poisson_loads(n, 8, seed).astype(np.uint64) + 45
    pin[n // 2] = 0
    pin_h = ones.copy()
    pin_h[n // 2] = 0
    big = (1 << 24) + rng.integers(0, 300, size=n).astype(np.uint64)
    return [("poisson", synth.poisson_loads(n, 8, seed).astype(np.uint64), ones), ("gate", gate, ones), ("pinned", pin, pin_h),
            ("big", big, ones)]


def _token_batches(n_batches, seed):
    seqs = synth.gen_sequences(200, T, seed)
    rng = np.random.default_rng(seed)
    out = []
    for b in range(n_batches):
        q = synth.gen_queries(seqs, B, seed * 100 + b, block=16)
        novel = rng.random(B) < 0.3
        q[novel] = rng.integers(0, 50000, size=(int(novel.sum()), T), dtype=np.uint32)
        out.append([list(map(int, r[: int(rng.integers(1, T + 1))])) for r in q])
    return out, seqs


TOPICS = ["Explain", "Summarise", "Translate to 中文:", "Write a haiku about", "Debug this code:", "List facts on", "Écris un poème sur", "🔥 Roast"]
SUBJECTS = ["radix trees", "memory systems", "load balancing", "cache-aware routing", "naïve café crème brûlée", "GPU 调度", "emoji 👋🌍"]


def _texts(n, seed):
    r = random.Random(seed)
    system = ["You are a helpful assistant.", "You are a terse assistant. Answer in one line.", ""]
    out = []
    for _ in range(n):
        if r.random() < 0.3:   # novel: nothing in the tree starts like it
            out.append("".join(r.choice("ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789") for _ in range(r.randrange(4, 40))))
            continue
        s = r.choice(system)
        body = f"{r.choice(TOPICS)} {r.choice(SUBJECTS)} {'x' * r.randrange(0, 40)} (variant {r.randrange(0, 50)})"
        out.append((s + " " + body) if s else body)
    return out


def _run(pol, ws, op, entry, reqs, loads, healthy, tag):
    n = len(ws)
    for w, l, h in zip(ws, loads, healthy):
        w.set_load(int(l)); w.set_healthy(bool(h))
    op.set_state(loads, healthy, [1] * n)
    if entry == "tokens":
        idx, info = pol.select_worker_batch(ws, reqs)
        want = FS.stream(op, loads, requests=reqs)
    elif entry == "request_text":
        idx, info = pol.select_worker_batch_request_text(ws, reqs)
        want = FS.stream(op, loads, texts=reqs)
    else:   # text in, token tree: the oracle routes the ids the device tokenizer produced
        idx, info, toks = pol.select_worker_batch_text(ws, reqs)
        want = FS.stream(op, loads, requests=toks)
    widx, wbr, wma, winp, wafter = want
    assert np.array_equal(idx, widx), (tag, int((idx != widx).sum()), int(np.argmax(idx != widx)))
    assert [i.branch for i in info] == list(wbr), tag
    assert [i.matched for i in info] == list(wma) and [i.input for i in info] == list(winp), tag
    after = np.asarray(loads, np.uint64) + np.bincount(idx[idx >= 0], minlength=n).astype(np.uint64)
    assert np.array_equal(after, wafter), tag
    return idx, np.asarray(wbr)


def _final_state(pol, op, kind):
    if kind == "text":
        assert pol.string_tree().entries() == op.string_tree().entries()     # nodes, tenants and epochs
    else:
        assert pol.token_tree().entries() == op.token_tree().entries()       # nodes, tenants and timestamps
    hk = "text" if kind == "text" else "tokens"
    want = op.hash_index(hk)
    assert pol.hash_index_size(hk) == len(want)
    for h, val in want.items():
        got = pol.hash_index_get(h, hk)
        assert got == (val if kind == "text" else list(val))


def _common_checks(fleet_name, idx, br, n):
    if fleet_name == "poisson":
        ml = br == FS.BR["tree_min_load"]
        assert ml.sum() > B // 10 and len(set(int(x) for x in idx[ml])) > 8     # the min-load picks spread over the fleet
    if fleet_name == "gate":
        im = br == FS.BR["imbalanced_min_load"]
        assert im[:60].all() and not im[64]                                      # open at the start, closed inside the batch
    if fleet_name == "pinned":
        assert n // 2 not in set(int(x) for x in idx)


@pytest.mark.parametrize("n_workers,empty_indexer", [(64, False), (256, False), (64, True)])
def test_token_tree_stream_matches_one_by_one_oracle(n_workers, empty_indexer):
    pol, ws, op = _pair(n_workers, empty_indexer=empty_indexer)
    batches, seqs = _token_batches(5, n_workers + 3)
    # a cached prefix whose tenant has left the slice: matching requests fall back to healthy[0], which is bumped without an insert
    pol.token_tree().insert_tokens(list(map(int, seqs[0])), GONE)
    op.token_tree().insert_tokens(list(map(int, seqs[0])), GONE)
    batches[0][:64] = [list(map(int, seqs[0]))] * 64
    falls = 0
    for b, (name, loads, healthy) in enumerate([("warm", np.zeros(n_workers, np.uint64), np.ones(n_workers, np.uint8))] + _fleets(n_workers, n_workers)):
        idx, br = _run(pol, ws, op, "tokens", batches[b], loads, healthy, (name, b))
        _common_checks(name, idx, br, n_workers)
        falls += int((br == FS.BR["tree_fallback_first_healthy"]).sum())
    assert falls > 0
    _final_state(pol, op, "tokens")
    assert list(pol.take_processed()) == [op.processed(i) for i in range(n_workers)]


@pytest.mark.parametrize("n_workers", [64, 256])
def test_string_tree_stream_matches_one_by_one_oracle(n_workers):
    pol, ws, op = _pair(n_workers)
    gone = "You are a helpful assistant. Explain radix trees in depth (cached by a worker that has left)"
    pol.string_tree().insert_text(gone, GONE)
    op.string_tree().insert_text(gone, GONE)
    falls = 0
    for b, (name, loads, healthy) in enumerate([("warm", np.zeros(n_workers, np.uint64), np.ones(n_workers, np.uint8))] + _fleets(n_workers, n_workers + 1)):
        texts = _texts(B, 1000 * n_workers + b)
        texts[: 40] = [gone] * 40 if b == 0 else texts[:40]
        idx, br = _run(pol, ws, op, "request_text", texts, loads, healthy, (name, b))
        _common_checks(name, idx, br, n_workers)
        falls += int((br == FS.BR["tree_fallback_first_healthy"]).sum())
    assert falls > 0
    _final_state(pol, op, "text")
    assert list(pol.take_processed()) == [op.processed(i) for i in range(n_workers)]


@pytest.mark.parametrize("n_workers", [64, 256])
def test_text_in_token_tree_stream_matches_one_by_one_oracle(n_workers):
    pol, ws, op = _pair(n_workers, tokenizer=True)
    for b, (name, loads, healthy) in enumerate([("warm", np.zeros(n_workers, np.uint64), np.ones(n_workers, np.uint8))] + _fleets(n_workers, n_workers + 2)):
        idx, br = _run(pol, ws, op, "text_in", _texts(B, 7000 * n_workers + b), loads, healthy, (name, b))
        _common_checks(name, idx, br, n_workers)
    _final_state(pol, op, "tokens")
    assert list(pol.take_processed()) == [op.processed(i) for i in range(n_workers)]


def test_relaunch_continues_from_the_running_loads():
    """X, X, Y with X and Y novel: the second X shares X's first page, so the walk restarts there after X's insert.  Loads 0, 1, 1, …: X goes
    to worker 0, the second X to its tenant, worker 0 again, and Y to worker 1 only if the restarted pass still counts the first X's bump
    (worker 0 at 2); a pass that started again from the snapshot would see worker 0 at 1 and, first among the minima, pick it."""
    pol, ws, op = _pair(8)
    loads, healthy = np.array([0] + [1] * 7, np.uint64), np.ones(8, np.uint8)
    distinct = [[7000 + 50 * i + k for k in range(40)] for i in range(3)]
    l0 = pol.kernel_launches()
    _run(pol, ws, op, "tokens", distinct, loads, healthy, "distinct")
    one = pol.kernel_launches() - l0
    x, y = [9000 + k for k in range(40)], [9500 + k for k in range(40)]
    l0 = pol.kernel_launches()
    idx, br = _run(pol, ws, op, "tokens", [x, x, y], loads, healthy, "dup")
    assert pol.kernel_launches() - l0 > one                # the second X was walked again
    assert list(idx) == [0, 0, 1]
    assert list(br) == [FS.BR["tree_min_load"], FS.BR["tree_match"], FS.BR["tree_min_load"]]
    _final_state(pol, op, "tokens")


def test_text_in_on_a_populated_event_index_with_an_imbalanced_snapshot_takes_the_event_stream():
    """Without feedback such a call detours through the token tree with the snapshot gate; with it the gate is per request, so the text-in
    call runs the event-driven stream — the same picks as the tokens-in call and as the oracle's one-by-one stream with bumps."""
    bs, n = 4, 16
    picks = []
    for entry in ("text_in", "tokens"):
        pol, ws, op = _pair(n)
        tok = pol.load_tiktoken_tokenizer(os.path.join(GOLD, "synth_vocab.tiktoken"), json.load(open(os.path.join(GOLD, "bpe_vectors.json")))["specials"])
        mon = pol.kv_event_monitor(bs)
        ix = mon.create_indexer("unknown", 8)
        mon.set_block_size("unknown", bs)
        pol.set_kv_event_monitor(mon)
        oix = orc.PositionalIndexer(8)
        op.attach_indexer("unknown", oix)
        op.set_block_size("unknown", bs)
        op.set_kv_event_monitor(True)
        for u in synth.worker_urls(n):
            assert ix.intern_worker(u) == oix.intern_worker(u)
        texts = _texts(400, 31)
        toks = tok.encode_batch(texts)
        seq = 1
        for k, t in enumerate(toks[:40]):
            hs = orc.compute_request_content_hashes(t, bs)
            blocks = [(seq + i, h) for i, h in enumerate(hs)]
            seq += len(blocks)
            if blocks:
                ix.apply_stored(k % n, blocks); oix.apply_stored(k % n, blocks)
        loads = np.full(n, 10, np.uint64)
        loads[3] = 90      # max - min = 80 > 64: open at the start, closed once the other 15 workers reach 26 (240 water-filling picks)
        for w, l in zip(ws, loads):
            w.set_load(int(l))
        op.set_state(loads, [1] * n, [1] * n)
        if entry == "text_in":
            idx, info, got = pol.select_worker_batch_text(ws, texts)
            assert got == toks
        else:
            idx, info = pol.select_worker_batch(ws, toks)
        flat = np.concatenate([np.asarray(t, np.uint32) for t in toks])
        offs = np.zeros(len(toks) + 1, np.uint64); np.cumsum([len(t) for t in toks], out=offs[1:])
        want, wbr, _, _ = op.select_batch_tokens_feedback(flat, offs)
        assert np.array_equal(idx, want), entry
        assert [i.branch for i in info] == list(wbr), entry
        assert (np.asarray(wbr) == 1).any() and (np.asarray(wbr) == 2).any()   # the gate was open, then closed inside the batch
        picks.append(idx)
    assert np.array_equal(picks[0], picks[1])


def test_frozen_batches_send_every_min_load_request_to_one_worker():
    pol, ws, op = _pair(64, feedback=False)
    loads, healthy = synth.poisson_loads(64, 8, 5).astype(np.uint64), np.ones(64, np.uint8)
    for w, l in zip(ws, loads):
        w.set_load(int(l))
    idx, info = pol.select_worker_batch_request_text(ws, _texts(B, 5))
    br = np.asarray([i.branch for i in info])
    assert (br == FS.BR["tree_min_load"]).sum() > 0 and len(set(int(x) for x in idx[br == FS.BR["tree_min_load"]])) == 1


def test_feedback_off_is_bit_equal_to_frozen_batches():
    """mask 0, and the event-only switch, leave tree-mode results exactly as they were."""
    runs = []
    for how in ("never", "mask0", "event_only"):
        pol, ws, op = _pair(64, feedback=False, tokenizer=True)
        if how == "mask0":
            pol.set_load_feedback_all_modes(True)
            pol._h.call("smgx_set_load_feedback_policies", 0)
        if how == "event_only":
            pol.set_load_feedback_all_modes(True)
            pol.set_load_feedback(True)
        out = []
        batches, _ = _token_batches(3, 11)
        for b, (name, loads, healthy) in enumerate(_fleets(64, 11)[:3]):
            for w, l, h in zip(ws, loads, healthy):
                w.set_load(int(l)); w.set_healthy(bool(h))
            i1, f1 = pol.select_worker_batch(ws, batches[b])
            i2, f2 = pol.select_worker_batch_request_text(ws, _texts(300, b))
            i3, f3, _ = pol.select_worker_batch_text(ws, _texts(300, 50 + b))
            out.append((i1.tolist(), [(x.branch, x.matched, x.input) for x in f1], i2.tolist(), [(x.branch, x.matched, x.input) for x in f2],
                        i3.tolist(), [(x.branch, x.matched, x.input) for x in f3]))
        out.append((pol.token_tree().entries(), pol.string_tree().entries(), list(pol.take_processed())))
        runs.append(out)
    assert runs[0] == runs[1] == runs[2]


def test_snapshot_tree_batch_mode_call_refuses_feedback():
    from smg_b200 import SmgxError, _lib
    pol, ws, op = _pair(8)
    pol.set_tree_batch_mode("snapshot")
    before = (pol.token_tree().entries(), pol.string_tree().entries())
    for call in (lambda: pol.select_worker_batch(ws, [[1, 2, 3]]), lambda: pol.select_worker_batch_request_text(ws, ["hello"])):
        with pytest.raises(SmgxError) as e:
            call()
        assert e.value.code == _lib.INVALID_ARGUMENT
    assert (pol.token_tree().entries(), pol.string_tree().entries()) == before
    pol.set_tree_batch_mode("sequential")
    _run(pol, ws, op, "request_text", ["hello"], np.zeros(8, np.uint64), np.ones(8, np.uint8), "after")
