"""Generates the golden fixtures of the Qwen2-family tokenizer.json (NFC normalizer + the single-digit Split).
Run from the repo root:  python tests/golden/gen_qwen2_golden.py

Source of truth, offline: the Python bindings of the `tokenizers` crate (the crate behind HuggingFaceTokenizer::encode).
Outputs (committed):  hf_qwen2_style_tokenizer.json  normalizer NFC, pre_tokenizer Split(Qwen2 regex, Isolated) + ByteLevel(use_regex=False),
                                                     a byte-level BPE trained here, added tokens <|endoftext|> <|im_start|> <|im_end|> <|K|>
                                                     (all normalized = false)
                      qwen2_vectors.json             texts + the ids `tokenizers` gives them with that fixture
"""
import json
import os
import random
import sys
import unicodedata

import tokenizers
from tokenizers import AddedToken, Regex, Tokenizer, decoders, models, normalizers, pre_tokenizers, trainers

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from smg_b200.policy import QWEN2_SPLIT_PATTERN  # noqa: E402

FIXTURE = "hf_qwen2_style_tokenizer.json"
SPECIALS = ["<|endoftext|>", "<|im_start|>", "<|im_end|>", "<|K|>"]
# marks that `tokenizers` gives class 0 although Unicode 15 does not (tools/gen_nfc_tables.py pins them), and the expanding code points
LATE_MARKS = "഻߽᷶\U0001e4efࣔ"
EXPANDING = "\U0001d160שּׁक़K;"

EDGES = [
    "12345", "a1b2c3", " 2024-10-15", "3.14159", "x=12+345", "１２３", "٣٤٥ ½",
    unicodedata.normalize("NFD", "naïve café déjà vu Ångström"), "Ångström", "ẹ́ ạ́ ớ",
    unicodedata.normalize("NFD", "한국어 텍스트 정규화"), "각 한", "한국어",
    "你好世界，今天天气怎么样？", "def f(x):\n    return x ** 2  # 42\n", "{\"key\": [1, 2, 3]}",
    EXPANDING, EXPANDING * 3, "\U0001d160" * 10, "a" + LATE_MARKS + "b", "क" + LATE_MARKS + "̴́",
    "<|im_start|>user\nhello<|im_end|>\n<|im_start|>assistant\n", "<|im_end|>́x", "<|im_start|>̣́",
    "<|K|>", "<|K|>", "<|K|><|K|>", "a<|K|>b<|K|>c", "<|endoftext|><|im_start|><|im_end|>", "<|endoftext|>",
    "e<|im_end|>́", "   ", "\n\n\n", "x \t y", "don't I'll we've they're IT'S",
    "x" + "́" * 300, "1" * 300, unicodedata.normalize("NFD", "é") * 150,
]


def corpus(n, seed):
    words = ("the quick brown fox jumps over lazy dog cache aware router prefix tree worker load balance token hello world "
             "naïve café crème brûlée déjà Ångström 你好 世界 调度 정규화 한국어 텍스트 été ça Straße größer 12345 2024 3.14159 don't "
             "I'll we've x=y+1 foo_bar() {\"key\": [1, 2, 3]} https://example.com/a?b=c&d=e \t tab\n newline\r\n crlf   spaces "
             "👋🌍 emoji ＡＢＣ ١٢٣ 's 'LL ṩ ệ ǖ").split(" ")
    r = random.Random(seed)
    out = []
    for _ in range(n):
        t = " ".join(r.choice(words) for _ in range(r.randrange(1, 40)))
        out.append(unicodedata.normalize("NFD", t) if r.random() < 0.3 else t)
    return out


def build_tokenizer(extra):
    tok = Tokenizer(models.BPE())
    tok.normalizer = normalizers.NFC()
    tok.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(QWEN2_SPLIT_PATTERN), behavior="isolated", invert=False),
                                                 pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=3000, special_tokens=[], initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False)
    tok.train_from_iterator(corpus(4000, 7) + extra, trainer)
    tok.add_special_tokens([AddedToken(s, special=True, normalized=False) for s in SPECIALS])
    return tok


def main():
    tok = build_tokenizer(EDGES)
    open(os.path.join(HERE, FIXTURE), "w").write(tok.to_str(pretty=False))
    saved = json.load(open(os.path.join(HERE, FIXTURE)))
    assert saved["normalizer"] == {"type": "NFC"}
    assert [a["normalized"] for a in saved["added_tokens"]] == [False] * len(SPECIALS)
    texts = corpus(30, 11) + EDGES
    ids = [e.ids for e in tok.encode_batch(texts, add_special_tokens=False)]
    json.dump({"generator": f"tokenizers {tokenizers.__version__}", "fixture": FIXTURE, "pattern": QWEN2_SPLIT_PATTERN,
               "cases": [{"text": t, "ids": i} for t, i in zip(texts, ids)]},
              open(os.path.join(HERE, "qwen2_vectors.json"), "w"), ensure_ascii=False)
    print("qwen2 texts", len(texts), "vocab", tok.get_vocab_size(), "tokens", sum(len(x) for x in ids))


if __name__ == "__main__":
    main()
