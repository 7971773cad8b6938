"""bench.py's text-in leg on its own, with the default sizes of bench.py:
    python tools/tokbench.py [cl100k_base|r50k_base|qwen2|qwen2-nonorm|llama2|deepseek] [--nfd]
cl100k_base / r50k_base pick the pre-tokenizer regex over the synthetic tiktoken vocabulary.  qwen2 loads the Qwen2-style tokenizer.json
fixture (NFC normalizer, single-digit Split); qwen2-nonorm the same file with its normalizer removed, so that the difference is the cost
of the NFC stage.  llama2 loads the Llama-2-style fixture (▁ normalization, byte fallback; a 1 210-entry vocabulary, not a real 32 000-entry
one) and deepseek the DeepSeek-V3-style fixture (the chain of three Splits; an 816-entry vocabulary, not DeepSeek's 128 000 entries); both
also time `tokenizers` encode_batch on the host threads over the corpus's first `batch` documents.  --nfd converts the corpus to NFD first,
so that every accented letter takes the normalizer's slow path.
Prints one JSON line."""
import functools, sys, os, json, tempfile, unicodedata
sys.path.insert(0, os.getcwd())
import bench
from smg_b200 import CacheAwarePolicy
enc = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("--") else "cl100k_base"
nfd = "--nfd" in sys.argv
FIXTURES = {"llama2": "hf_llama2_style_tokenizer.json", "deepseek": "hf_deepseek_v3_style_tokenizer.json"}
if enc.startswith("qwen2") or enc in FIXTURES:
    fixture = os.path.join(os.getcwd(), "tests", "golden", FIXTURES.get(enc, "hf_qwen2_style_tokenizer.json"))
    if enc == "qwen2-nonorm":
        j = json.load(open(fixture))
        j["normalizer"] = None
        fixture = os.path.join(tempfile.mkdtemp(), "qwen2_nonorm.json")
        json.dump(j, open(fixture, "w"))
    CacheAwarePolicy.load_tiktoken_tokenizer = lambda self, path, special_tokens=None, model="unknown", **kw: self.load_hf_tokenizer(fixture, model)
else:
    CacheAwarePolicy.load_tiktoken_tokenizer = functools.partialmethod(CacheAwarePolicy.load_tiktoken_tokenizer, encoding=enc)
_docs, corpus = bench.text_corpus_docs, []
def _corpus_docs(*a, **kw):
    docs, lines = _docs(*a, **kw)
    if nfd:
        docs, lines = [unicodedata.normalize("NFD", d) for d in docs], [unicodedata.normalize("NFD", x) for x in lines]
    corpus.extend(docs)
    return docs, lines
bench.text_corpus_docs = _corpus_docs
class A: pass
a=A(); a.batch=4096; a.workers=64; a.text_docs=8192; a.text_bytes=2048; a.steps=2000
res = bench.text_in_leg(a, 0)
res.pop("cpu_tokenize_baseline", None)   # always measured with the cl100k regex there
if enc in FIXTURES:
    import time, tokenizers
    ref, texts = tokenizers.Tokenizer.from_file(fixture), corpus[:a.batch]
    ref.encode_batch(texts[:256], add_special_tokens=False)
    t0 = time.perf_counter()
    ids = ref.encode_batch(texts, add_special_tokens=False)
    dt = time.perf_counter() - t0
    res["cpu_tokenize_baseline"] = {"value": len(texts) / dt, "unit": "requests/s", "tokens_per_s": sum(len(e.ids) for e in ids) / dt,
                                    "cores": os.cpu_count(), "kind": f"tokenizers {tokenizers.__version__} encode_batch, tokenize step only"}
print(json.dumps(dict(res, encoding=enc, nfd=nfd)))
