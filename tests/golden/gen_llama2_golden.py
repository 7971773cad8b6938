"""Generates the golden fixtures of the SentencePiece-style BPE tokenizer.json family (Llama 2, Mistral, TinyLlama, CodeLlama).
Run from the repo root:  python tests/golden/gen_llama2_golden.py

Source of truth, offline: the Python bindings of the `tokenizers` crate (the crate behind HuggingFaceTokenizer::encode).
Outputs (committed):  hf_llama2_style_tokenizer.json  shape (A): normalizer Sequence[Prepend("▁"), Replace(" " → "▁")], pre_tokenizer null,
                                                      a BPE with byte_fallback trained here whose vocabulary holds ▁word pieces, whitespace
                                                      runs (▁▁, ▁▁▁▁), accented letters and some CJK, and the 256 <0xXX> byte tokens as
                                                      plain vocab entries; added tokens <unk> <s> </s> <|user|> <|assistant|>
                                                      (all normalized = false)
                      llama2_vectors.json             texts + the ids `tokenizers` gives them, for shape (A) and for shape (B) — the same
                                                      model with normalizer null and pre_tokenizer Metaspace — with (prepend_scheme, split)
                                                      = (first, false), (always, false), (first, true)
The BPE is trained on text cut the way the GPU path cuts a stretch (before every ▁ that follows another character), so no merge joins a
piece ending in a non-▁ character to one starting with ▁ and the fixture passes the loader's exactness check.  Emoji, tabs, newlines and
some CJK never occur in the training text: they go through byte fallback.
"""
import json
import os
import random

import tokenizers
from tokenizers import Regex, Tokenizer, models, normalizers, pre_tokenizers, trainers

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = "hf_llama2_style_tokenizer.json"
SPECIALS = ["<unk>", "<s>", "</s>"]
CHAT = ["<|user|>", "<|assistant|>"]
LEGACY_NORMALIZER = {"type": "Sequence", "normalizers": [{"type": "Prepend", "prepend": "▁"},
                                                         {"type": "Replace", "pattern": {"String": " "}, "content": "▁"}]}
# shape (B) variants: (prepend_scheme, split)
METASPACE_VARIANTS = [("first", False), ("always", False), ("first", True)]

WORDS = ("the quick brown fox jumps over lazy dog cache aware router prefix tree worker load balance token hello world "
         "a an of to in is it that this for with on as are be by at from or not have has was were will would could should "
         "naïve café crème brûlée déjà vu Ångström été ça Straße größer über señor niño façade "
         "你好 世界 今天 天气 中文 测试 数据 模型 "
         "def return if else for while import class self None True False x=y+1 foo_bar() {\"key\": [1, 2, 3]} 12345 2024 3.14159 "
         "don't I'll we've they're").split(" ")


def corpus(n, seed):
    r = random.Random(seed)
    out = []
    for _ in range(n):
        words = [r.choice(WORDS) for _ in range(r.randrange(1, 30))]
        sep = [" " * r.choice((1, 1, 1, 1, 2, 4, 8)) for _ in words]
        out.append("".join(s + w for s, w in zip(sep, words)).lstrip(" ") if r.random() < 0.7 else "".join(s + w for s, w in zip(sep, words)))
    return out


def build_json():
    """Train on text normalized as shape (A) does and cut before every ▁ that follows another character; then lay the vocabulary out as
    Llama 2 does: <unk> <s> </s>, the 256 byte tokens, the trained pieces."""
    tok = Tokenizer(models.BPE())
    tok.normalizer = normalizers.Sequence([normalizers.Prepend("▁"), normalizers.Replace(" ", "▁")])
    tok.pre_tokenizer = pre_tokenizers.Split(Regex("▁*[^▁]+|▁+"), behavior="isolated", invert=False)
    tok.train_from_iterator(corpus(6000, 7), trainers.BpeTrainer(vocab_size=1500, special_tokens=[], show_progress=False))
    trained = json.loads(tok.to_str())["model"]
    vocab = {s: i for i, s in enumerate(SPECIALS)}
    vocab.update({f"<0x{b:02X}>": 3 + b for b in range(256)})
    for s, _ in sorted(trained["vocab"].items(), key=lambda kv: kv[1]):
        vocab[s] = len(vocab)
    added = [{"id": vocab[s], "content": s, "single_word": False, "lstrip": False, "rstrip": False, "normalized": False, "special": True}
             for s in SPECIALS]
    added += [{"id": len(vocab) + k, "content": s, "single_word": False, "lstrip": False, "rstrip": False, "normalized": False, "special": True}
              for k, s in enumerate(CHAT)]
    return {
        "version": "1.0", "truncation": None, "padding": None, "added_tokens": added,
        "normalizer": LEGACY_NORMALIZER, "pre_tokenizer": None, "post_processor": None,
        "decoder": {"type": "Sequence", "decoders": [{"type": "Replace", "pattern": {"String": "▁"}, "content": " "}, {"type": "ByteFallback"},
                                                     {"type": "Fuse"}, {"type": "Strip", "content": " ", "start": 1, "stop": 0}]},
        "model": {"type": "BPE", "dropout": None, "unk_token": "<unk>", "continuing_subword_prefix": None, "end_of_word_suffix": None,
                  "fuse_unk": True, "byte_fallback": True, "ignore_merges": False, "vocab": vocab, "merges": trained["merges"]},
    }


def metaspace(j, prepend_scheme, split):
    """Shape (B): the same model with the ▁ rule moved from the normalizer into a Metaspace pre-tokenizer."""
    j = json.loads(json.dumps(j))
    j["normalizer"] = None
    j["pre_tokenizer"] = {"type": "Metaspace", "replacement": "▁", "prepend_scheme": prepend_scheme, "split": split}
    return j


def texts():
    cjk_long = "你好世界今天天气中文测试数据模型龍鳳麒麟" * 20          # 400 code points, no space; the last four fall back to bytes
    edges = [
        "", " ", "   ", " leading", "trailing ", "double  space", "  both  ", "a", "▁", "▁▁x", "a▁b", " ▁x", "x ▁", "literal <0x41> and <0x0A>",
        "<s>", "<s> hello", "<s>hello</s>", "hello </s>", "<s></s>", "<s><|user|></s>", "</s> ", " <s> ", "<unk>", "x<unk>y",
        "<|user|>\nhow are you?</s>\n<|assistant|>\n I am fine.</s>", "<|user|> <|assistant|>",
        "tab\there", "\t\tindented", "line one\nline two", "crlf\r\nline", "\n", "\r\n", " \n ",
        "emoji 👋🌍🎉", "👋👋👋👋", "🧑‍💻 coder", "x🎉y", "mixed 中文 and English 😀",
        "naïve café (NFD, no NFC here)", "é vs é", "Ångström Ångström",
        cjk_long, "龍" * 300, " " + cjk_long + " end", "a" * 14, "a" * 15, "a" * 16, "x" * 31, "x" * 32, "x" * 33,
        "y" * 255, "y" * 256, "y" * 257, "z" * 600, " " * 40, " " * 300, "    def f(self):\n        return None  # indent",
        "The quick brown fox jumps over the lazy dog. The router is cache aware: it keeps a prefix tree per worker and sends each "
        "request to the worker that already holds the longest prefix, unless the load is unbalanced.",
        "Hey 👋 how's it going? 🚀🔥 Let's test: ünïcödé, 日本語, 한국어, عربي, and some ≠ ≤ ≥ math ∑∫√ and more 🎉🎊🥳!",
        "1234567890 3.14159 x=y+1 foo_bar() {\"key\": [1, 2, 3]}",
    ]
    r = random.Random(11)
    return corpus(30, 11) + edges + ["".join(r.choice(["▁", " ", "a", "é", "中", "😀", "\t", "<s>", "</s>", "bc", "  "])
                                         for _ in range(r.randrange(0, 40))) for _ in range(40)]


def encode(j, ts):
    tk = Tokenizer.from_str(json.dumps(j))
    return [e.ids for e in tk.encode_batch(ts, add_special_tokens=False)]


def main():
    j = build_json()
    open(os.path.join(HERE, FIXTURE), "w").write(json.dumps(j, ensure_ascii=False))
    ts = texts()
    out = {"generator": f"tokenizers {tokenizers.__version__}", "fixture": FIXTURE, "cases": [{"text": t} for t in ts], "variants": {}}
    out["variants"]["legacy"] = encode(j, ts)
    for ps, sp in METASPACE_VARIANTS:
        out["variants"][f"metaspace-{ps}-{'split' if sp else 'nosplit'}"] = encode(metaspace(j, ps, sp), ts)
    json.dump(out, open(os.path.join(HERE, "llama2_vectors.json"), "w"), ensure_ascii=False)
    print("llama2 texts", len(ts), "vocab", len(j["model"]["vocab"]), "merges", len(j["model"]["merges"]),
          "tokens", sum(len(x) for x in out["variants"]["legacy"]))


if __name__ == "__main__":
    main()
