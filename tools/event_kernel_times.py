#!/usr/bin/env python
"""Where the time of bench.py's event-driven pick goes, kernel by kernel.

    python tools/event_kernel_times.py OUT_DIR [--steps 2000,20]

Builds bench.py's config-2 workload with its own helpers (64 workers, 1.0 M-entry index, a ring of 4096-request batches of 512
tokens), issues bench.py's call shape (K batches handed to smgx_select_many_tokens_device in one call, spread over the stream lanes)
once unprofiled to warm up and once under torch.profiler with CUDA activities, writes the trace to OUT_DIR/trace_k{K}.json and prints
one JSON line per K: per kernel name the launches, total and mean time, decisions per kernel-second and the modelled bytes per
kernel-second, then the span of the call on the GPU, the time any kernel ran and the idle time between them.

Bytes model (what the default kernel requests per decision, not DRAM traffic: the probes mostly hit L2): 8 B of offsets, 4 B of pick,
64 B of tokens for each block hashed and 32 B per lookup.  A full hit or a novel request hashes blocks 0 and last and probes their
slots.  A failed count test drains positions 1..last-1 in segments of 8 and stops at the segment holding the first missing position (a
partial hit keeps k whole blocks, so position k): it hashes blocks 0, last and every position of the segments it reads, and reads the
32 B run-arena record of each drained position (contiguous records from the anchor of block 0's entry) in place of its slot; a
position whose record misses (the missing one, or a run broken by another store) adds a 1 B tag and, where the tag matches, a slot,
which this model does not count.
Profile in a run of its own: tracing slows the host, so these times are not the bench's.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def bytes_per_decision(kinds, keeps, T, bs):
    """Mean modelled bytes per decision over the ring (kinds: 0 full hit, 1 partial → failed count test, 2 novel; keeps: tokens a
    partial hit keeps)."""
    last = T // bs - 1
    stop = np.clip(keeps // bs, 1, last)                                   # the drain's first missing position
    drained = np.minimum(8 * ((stop - 1) // 8 + 1), last - 1)             # whole segments of 8 up to it, within 1..last-1
    blocks = np.where(kinds == 1, 2 + drained, 2)                        # each: 64 B of tokens + a 32 B slot (0, last) or record (drained)
    return float((8 + 4 + blocks * (4 * bs + 32)).mean())


def union_us(spans):
    busy, end = 0.0, -np.inf
    for s, e in sorted(spans):
        if e > end:
            busy += e - max(s, end)
            end = e
    return busy


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--steps", default="2000,20", help="comma-separated K: batches per smgx_select_many_tokens_device call")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--tokens", type=int, default=512)
    ap.add_argument("--workers", type=int, default=64)
    ap.add_argument("--sequences", type=int, default=31250)
    ap.add_argument("--ring", type=int, default=32)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile

    from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy, synth
    from smg_b200 import _lib
    B, T, W, bs, R = args.batch, args.tokens, args.workers, 16, args.ring
    torch.cuda.init()
    pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, **bench.CFG), device_id=0, max_batch=B, max_tokens_per_request=T)
    h, L = pol._h, _lib.load()
    ws = [BasicWorker(u) for u in synth.worker_urls(W)]
    for w, ld in zip(ws, synth.poisson_loads(W, 8, 42)):
        w.set_load(int(ld))
    pol.init_workers(ws)
    mon = pol.kv_event_monitor(bs)
    ix = mon.create_indexer("unknown", 64)
    pol.set_kv_event_monitor(mon)
    seqs = bench.build_population(args.sequences, T, 42)
    bench.populate(pol, ix, seqs, W, bs)
    model = pol._push_fleet(ws)

    err = _lib.new_err()
    offsets = (np.arange(B + 1, dtype=np.uint64) * T).astype(np.uint32)
    d_off = L.smgx_device_alloc(h.p, offsets.nbytes, C.byref(err))
    h.call("smgx_memcpy_h2d", d_off, offsets.ctypes.data_as(C.c_void_p), offsets.nbytes)
    d_tok, d_out, kinds_all, keeps_all = [], [], [], []
    for r in range(R):
        q, kinds, keeps = bench.gen_batch(seqs, B, 42 + r, bs)
        kinds_all.append(kinds); keeps_all.append(keeps)
        flat = np.ascontiguousarray(q.reshape(-1))
        dt = L.smgx_device_alloc(h.p, flat.nbytes, C.byref(err))
        h.call("smgx_memcpy_h2d", dt, flat.ctypes.data_as(C.c_void_p), flat.nbytes)
        d_tok.append(dt)
        d_out.append(L.smgx_device_alloc(h.p, B * 4, C.byref(err)))
    model_bytes = bytes_per_decision(np.concatenate(kinds_all), np.concatenate(keeps_all), T, bs)

    for K in [int(k) for k in args.steps.split(",")]:
        order = [i % R for i in range(K)]
        TOK = (C.c_void_p * K)(*[d_tok[j] for j in order])
        OFF = (C.c_void_p * K)(*[d_off] * K)
        OUT = (C.c_void_p * K)(*[d_out[j] for j in order])
        NS = (C.c_uint32 * K)(*[B] * K)
        h.call("smgx_select_many_tokens_device", model, K, TOK, OFF, NS, T, OUT)   # warm-up: scratch allocations, module load
        h.call("smgx_synchronize")
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            h.call("smgx_select_many_tokens_device", model, K, TOK, OFF, NS, T, OUT)
            h.call("smgx_synchronize")
        trace = os.path.join(args.out, f"trace_k{K}.json")
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            events = json.load(f)["traceEvents"]
        kern = [e for e in events if e.get("cat") == "kernel" and "dur" in e]
        decisions = K * B
        per = {}
        for e in kern:
            p = per.setdefault(e["name"], {"launches": 0, "total_us": 0.0})
            p["launches"] += 1
            p["total_us"] += float(e["dur"])
        for p in per.values():
            p["mean_us"] = p["total_us"] / p["launches"]
            p["decisions_per_kernel_s"] = decisions / (p["total_us"] * 1e-6)
            p["model_GBps"] = model_bytes * decisions / (p["total_us"] * 1e-6) / 1e9
        spans = [(float(e["ts"]), float(e["ts"]) + float(e["dur"])) for e in kern]
        span = (max(e for _, e in spans) - min(s for s, _ in spans)) if spans else 0.0
        busy = union_us(spans)
        print(json.dumps({"steps": K, "decisions": decisions, "model_bytes_per_decision": model_bytes, "kernels": per,
                          "span_us": span, "any_kernel_running_us": busy, "idle_us": span - busy,
                          "decisions_per_span_s": decisions / (span * 1e-6) if span else None, "trace": trace}), flush=True)
    for dptr in d_tok + d_out + [d_off]:
        L.smgx_device_free(h.p, dptr)


if __name__ == "__main__":
    main()
