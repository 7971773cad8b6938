"""Generates tests/golden/consistent_hashing_vectors.json: key positions blake3(key)[..8] (LE) for keys of 0 bytes to several blake3
chunks, and whole consistent_hashing decisions without a ring (model_gateway/src/policies/consistent_hashing.rs:68-111: the healthy
URL → last healthy index map, its values sorted, position % len), restated in plain Python on top of the independent `blake3` package
(bindings of the official Rust crate).  It pins the oracle (tests/consistent_hashing_oracle.py) and the CUDA path.
Run from the repo root: python tests/golden/gen_consistent_hashing_golden.py"""
import json
import os
import random

import blake3

# one chunk is 1024 bytes, one group of the long-key kernel 32 chunks
LENGTHS = [0, 1, 63, 64, 65, 1023, 1024, 1025, 2048, 3073, 8192 + 17, 32 * 1024, 32 * 1024 + 1, 33 * 1024, 40 * 1024 - 3, 64 * 1024 + 5,
           100_000, 300_000]


def key_bytes(n: int, salt: int) -> bytes:   # visible ASCII, so every key is also a valid header value
    return bytes(0x21 + (i * 7 + salt * 13 + (i >> 10)) % 94 for i in range(n))


def position(b: bytes) -> int:
    return int.from_bytes(blake3.blake3(b).digest()[:8], "little")


def main():
    keys = [{"len": n, "salt": s, "pos": str(position(key_bytes(n, s)))} for n in LENGTHS for s in (0, 1)]
    rng = random.Random(20261018)
    decisions = []
    for case in range(8):
        w = rng.choice([1, 2, 3, 5, 17, 64])
        urls = [f"http://w{rng.randrange(max(1, w - 2))}:8000" if rng.random() < 0.2 else f"http://worker-{i}:8000" for i in range(w)]
        healthy = [1 if rng.random() < 0.8 else 0 for _ in range(w)]
        last = {}
        for i, u in enumerate(urls):
            if healthy[i]:
                last[u] = i
        vals = sorted(last.values())
        reqs = []
        for r in range(24):
            n, salt = rng.choice([1, 36, 200, 1500, 5000]), case * 100 + r
            kp = position(key_bytes(n, salt))
            reqs.append({"len": n, "salt": salt, "pos": str(kp), "idx": vals[kp % len(vals)] if vals else -1})
        decisions.append({"urls": urls, "healthy": healthy, "requests": reqs})
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "consistent_hashing_vectors.json")
    with open(out, "w") as f:
        json.dump({"keys": keys, "no_ring_decisions": decisions}, f, indent=0)
        f.write("\n")
    print(out)


if __name__ == "__main__":
    main()
