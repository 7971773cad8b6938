"""Cost of load feedback in the tree modes: a tree-mode batch with SMGX_FEEDBACK_CACHE_AWARE against the same batch decided against one
frozen fleet snapshot.  Both are synchronous calls (H2D, walk kernels, host in-order pass, D2H), so a host clock around each call measures
the whole call.  The two variants run alternately on twin policies fed the same batches, so that both trees grow alike.

    python tools/feedback_cost.py [--workers 64] [--batch 4096] [--reps 20]

Prints the card name and power limit with the numbers."""
import argparse
import os
import random
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001 — the numbers are still printed, with the reason the card is unknown
        return f"unknown ({e})"


def texts(n, seed):
    r = random.Random(seed)
    system = ["You are a helpful assistant. " * 4, "You are a terse assistant. Answer in one line. " * 3, ""]
    out = []
    for _ in range(n):
        if r.random() < 0.3:
            out.append("".join(r.choice("ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789") for _ in range(r.randrange(16, 200))))
        else:
            out.append(r.choice(system) + f"question {r.randrange(0, 400)} " + "x" * r.randrange(0, 300))
    return out


def main():
    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy, synth
    ap = argparse.ArgumentParser()
    ap.add_argument("--workers", type=int, default=64)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    cfg = CacheAwareConfig(eviction_interval_secs=0, cache_threshold=0.5, balance_abs_threshold=32, balance_rel_threshold=1.1)
    urls = synth.worker_urls(a.workers)
    pols = {}
    for mode in ("frozen", "feedback"):
        pol = CacheAwarePolicy(cfg, max_batch=max(a.batch, 1))
        ws = [BasicWorker(u) for u in urls]
        pol.init_workers(ws)
        if mode == "feedback":
            pol.set_load_feedback_all_modes(True)
        loads = synth.poisson_loads(a.workers, 8, 1)
        for w, l in zip(ws, loads):
            w.set_load(int(l))
        pols[mode] = (pol, ws)
    batches = [texts(a.batch, s) for s in range(a.reps + 2)]
    for mode, (pol, ws) in pols.items():   # warm-up: first launches, tree growth of the first batches
        pol.select_worker_batch_request_text(ws, batches[0], want_info=False)
    ms = {"frozen": [], "feedback": []}
    for b in batches[1:]:
        for mode in ("frozen", "feedback"):
            pol, ws = pols[mode]
            t0 = time.perf_counter()
            pol.select_worker_batch_request_text(ws, b, want_info=False)
            ms[mode].append((time.perf_counter() - t0) * 1e3)
    print(f"card: {card()}")
    print(f"string tree, {a.workers} workers, {a.batch} requests per call, {len(ms['frozen'])} calls each, alternating")
    for mode, v in ms.items():
        v = np.asarray(v[1:])
        print(f"  {mode:9s} median {np.median(v):8.2f} ms   min {v.min():8.2f} ms   max {v.max():8.2f} ms")


if __name__ == "__main__":
    main()
