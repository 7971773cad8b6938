"""bench.py's text-in leg on its own, with the default sizes of bench.py:  python tools/tokbench.py [cl100k_base|r50k_base]
The argument picks the tokenizer's pre-tokenizer regex (same synthetic vocabulary).  Prints one JSON line."""
import functools, sys, os, json
sys.path.insert(0, os.getcwd())
import bench
from smg_b200 import CacheAwarePolicy
enc = sys.argv[1] if len(sys.argv) > 1 else "cl100k_base"
CacheAwarePolicy.load_tiktoken_tokenizer = functools.partialmethod(CacheAwarePolicy.load_tiktoken_tokenizer, encoding=enc)
class A: pass
a=A(); a.batch=4096; a.workers=64; a.text_docs=8192; a.text_bytes=2048; a.steps=2000
res = bench.text_in_leg(a, 0)
res.pop("cpu_tokenize_baseline", None)   # always measured with the cl100k regex there
print(json.dumps(dict(res, encoding=enc)))
