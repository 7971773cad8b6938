"""Builds the smgx shared library (hand-written sm_90a CUDA + the C ABI) in-tree: smg_b200/libsmgx.so.

nvcc cross-compiles for sm_90a without a GPU.  The .so is git-ignored; build() (or the test session) rebuilds it when a source is newer.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsmgx.so")
SOURCES = ["smgx.cu", "event_index.cu", "event_kernels.cu", "tokenizer.cu", "token_tree.cu", "string_tree.cu", "blake3.cu", "prefix_hash.cu", "power_of_two.cu", "consistent_hashing.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CFLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--fmad=false",            # f32 imbalance / match-rate compares must not be contracted (cache_aware.rs:670, :851)
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function,-Wno-unknown-pragmas",
]
LFLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-Xcompiler", "-fPIC"]
OBJDIR = os.path.join(HERE, "build")


def _deps():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "smgx.h"), __file__]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in _deps())


def _compile(src, obj, verbose):
    cmd = [NVCC] + CFLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src]
    res = subprocess.run(cmd, capture_output=True, text=True)
    return src, res


def build(force=False, verbose=False):
    """Every .cu is compiled to its own object in parallel (one nvcc process each), then linked; an object is reused when it is
    newer than every header and its own source."""
    if not force and not needs_build():
        return OUT
    from concurrent.futures import ThreadPoolExecutor
    os.makedirs(OBJDIR, exist_ok=True)
    hdr_t = max(os.path.getmtime(d) for d in _deps() if not d.endswith(".cu"))
    jobs, objs = [], []
    for s in SOURCES:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJDIR, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or verbose or not os.path.exists(obj) or os.path.getmtime(obj) < max(hdr_t, os.path.getmtime(src)):
            jobs.append((src, obj))
    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        for src, res in ex.map(lambda j: _compile(j[0], j[1], verbose), jobs):
            if res.returncode != 0:
                sys.stderr.write(res.stdout + res.stderr)
                raise RuntimeError("nvcc failed compiling " + src)
            if verbose or res.stderr.strip():
                sys.stderr.write(res.stdout + res.stderr)
    res = subprocess.run([NVCC] + LFLAGS + ["-o", OUT] + objs, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed linking libsmgx.so")
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(OUT)
