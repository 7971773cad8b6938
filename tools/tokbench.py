"""bench.py's text-in leg on its own, with the default sizes of bench.py:
    python tools/tokbench.py [cl100k_base|r50k_base|qwen2|qwen2-nonorm] [--nfd]
cl100k_base / r50k_base pick the pre-tokenizer regex over the synthetic tiktoken vocabulary.  qwen2 loads the Qwen2-style tokenizer.json
fixture (NFC normalizer, single-digit Split); qwen2-nonorm the same file with its normalizer removed, so that the difference is the cost
of the NFC stage.  --nfd converts the corpus to NFD first, so that every accented letter takes the normalizer's slow path.
Prints one JSON line."""
import functools, sys, os, json, tempfile, unicodedata
sys.path.insert(0, os.getcwd())
import bench
from smg_b200 import CacheAwarePolicy
enc = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("--") else "cl100k_base"
nfd = "--nfd" in sys.argv
if enc.startswith("qwen2"):
    fixture = os.path.join(os.getcwd(), "tests", "golden", "hf_qwen2_style_tokenizer.json")
    if enc == "qwen2-nonorm":
        j = json.load(open(fixture))
        j["normalizer"] = None
        fixture = os.path.join(tempfile.mkdtemp(), "qwen2_nonorm.json")
        json.dump(j, open(fixture, "w"))
    CacheAwarePolicy.load_tiktoken_tokenizer = lambda self, path, special_tokens=None, model="unknown", **kw: self.load_hf_tokenizer(fixture, model)
else:
    CacheAwarePolicy.load_tiktoken_tokenizer = functools.partialmethod(CacheAwarePolicy.load_tiktoken_tokenizer, encoding=enc)
if nfd:
    _docs = bench.text_corpus_docs
    def _nfd_docs(*a, **kw):
        docs, lines = _docs(*a, **kw)
        return [unicodedata.normalize("NFD", d) for d in docs], [unicodedata.normalize("NFD", x) for x in lines]
    bench.text_corpus_docs = _nfd_docs
class A: pass
a=A(); a.batch=4096; a.workers=64; a.text_docs=8192; a.text_bytes=2048; a.steps=2000
res = bench.text_in_leg(a, 0)
res.pop("cpu_tokenize_baseline", None)   # always measured with the cl100k regex there
print(json.dumps(dict(res, encoding=enc, nfd=nfd)))
