"""consistent_hashing on the GPU: kernel time, host-buffer request rate and a CPU baseline, on 64 workers with a ring and batches of 4096.

Request mix: 60 % X-SMG-Routing-Key of 36 bytes (a UUID), 20 % a ~200-byte bearer authorization, 10 % a cookie of 1-8 KB, 5 % an
X-SMG-Target-Worker, 5 % no headers.  Kernel time is the sum of the policy's kernels in a torch.profiler run of its own; the host-buffer
rate is end-to-end smgx_consistent_hashing_select_batch calls (copies and synchronisation included); the CPU baseline is the C++
restatement (tests/cpp/consistent_hashing_oracle.h) deciding the same batches on one host thread and on every host thread.  The card's name and power limit are read in the same run.
Usage: python tools/consistent_hashing_bench.py [--batches 200] [--out DIR]   (prints one JSON line)"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_batch(rng, n, w):
    hs = []
    for _ in range(n):
        u = rng.random()
        if u < 0.60:
            hs.append({"x-smg-routing-key": "%08x-%04x-%04x-%04x-%012x" % tuple(int(rng.integers(0, 2**b)) for b in (32, 16, 16, 16, 48))})
        elif u < 0.80:
            hs.append({"authorization": "Bearer " + "".join(chr(0x41 + int(c)) for c in rng.integers(0, 26, 193))})
        elif u < 0.90:
            hs.append({"cookie": "s=" + "".join(chr(0x61 + int(c)) for c in rng.integers(0, 26, int(rng.integers(1024, 8192))))})
        elif u < 0.95:
            hs.append({"x-smg-target-worker": str(int(rng.integers(0, w)))})
        else:
            hs.append(None)
    return hs


def pack(hs):
    from smg_b200.policy import _ch_header_values
    blob, offs, present = bytearray(), [0], []
    for hd in hs:
        bits = 0
        for h, v in enumerate(_ch_header_values(hd)):
            if v is not None:
                bits |= 1 << h
                blob += v
            offs.append(len(blob))
        present.append(bits)
    return bytes(blob), offs, present


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=200)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--workers", type=int, default=64)
    ap.add_argument("--out", default=None, help="directory for the profiler trace (default: none written)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    from smg_b200 import BasicWorker, ConsistentHashingPolicy
    from tests import consistent_hashing_oracle as ch

    rng = np.random.default_rng(2026)
    urls = [f"http://worker-{i}:8000" for i in range(args.workers)]
    ws = [BasicWorker(u) for u in urls]
    pol = ConsistentHashingPolicy(max_batch=args.batch)
    ring = pol.hash_ring(urls)
    batches = [pack(make_batch(rng, args.batch, args.workers)) for _ in range(8)]
    call = lambda k, s: pol.select_worker_batch(ws, ring=ring, seed=s, values=batches[k][0], offsets=batches[k][1], present=batches[k][2])  # noqa: E731
    for k in range(len(batches)):
        call(k, k)
    # host-buffer rate
    t0 = time.perf_counter()
    for s in range(args.batches):
        call(s % len(batches), s)
    host_s = time.perf_counter() - t0
    # kernel time, in a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(args.batches):
            call(s % len(batches), s)
    kern_us = {}
    for e in prof.key_averages():
        m = re.search(r"chash_\w+", e.key)
        if m:
            kern_us[m.group(0)] = kern_us.get(m.group(0), 0.0) + (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.out, "consistent_hashing.pt.trace.json"))
    # CPU baseline: the C++ oracle (tests/cpp/consistent_hashing_oracle.h) on host threads, same batches and seeds
    threads = os.cpu_count() or 1
    cpu = {}
    for t in sorted({1, threads}):
        ch.cpp_select_batch(urls, [1] * args.workers, urls, *batches[0], 0, t)   # warm-up
        secs = 0.0
        for k in range(len(batches)):
            secs += ch.cpp_select_batch(urls, [1] * args.workers, urls, *batches[k], k, t)[3]
        cpu[str(t)] = round(len(batches) * args.batch / secs)
    n_req = args.batches * args.batch
    print(json.dumps({
        "card": card, "workers": args.workers, "batch": args.batch, "batches": args.batches,
        "kernel_us_per_batch": {k: round(v / args.batches, 2) for k, v in kern_us.items()},
        "host_buffer_requests_per_s": round(n_req / host_s),
        "host_buffer_us_per_batch": round(host_s / args.batches * 1e6, 1),
        "cpu_baseline": "C++ oracle tests/cpp/consistent_hashing_oracle.h, requests split over host threads, decision time only",
        "cpu_baseline_requests_per_s_by_threads": cpu,
    }))


if __name__ == "__main__":
    main()
