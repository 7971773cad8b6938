"""Generates the golden fixtures of the DeepSeek-V3-family tokenizer.json (the chain of three Split pre-tokenizers).
Run from the repo root:  python tests/golden/gen_deepseek_golden.py

Source of truth, offline: the Python bindings of the `tokenizers` crate (the crate behind HuggingFaceTokenizer::encode).
Outputs (committed):  hf_deepseek_v3_style_tokenizer.json  normalizer Sequence[] (the identity), pre_tokenizer Sequence[Split(\\p{N}{1,3}),
                                                           Split(kana/CJK), Split(DeepSeek word regex), ByteLevel(use_regex=False)], all
                                                           Isolated; a byte-level BPE trained here; DeepSeek's multi-byte added tokens
                                                           <｜begin▁of▁sentence｜> <｜end▁of▁sentence｜> <｜User｜> <｜Assistant｜>
                      deepseek_vectors.json                texts + the ids `tokenizers` gives them with that fixture
"""
import json
import os
import random
import sys

import tokenizers
from tokenizers import AddedToken, Regex, Tokenizer, decoders, models, normalizers, pre_tokenizers, trainers

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from smg_b200.policy import DEEPSEEK_SPLIT_PATTERNS  # noqa: E402

FIXTURE = "hf_deepseek_v3_style_tokenizer.json"
BOS, EOS, USER, ASSISTANT = "<｜begin▁of▁sentence｜>", "<｜end▁of▁sentence｜>", "<｜User｜>", "<｜Assistant｜>"
SPECIALS = [BOS, EOS, USER, ASSISTANT]

EDGES = [
    # digit runs of length 1-10, ASCII and other scripts
    *["1234567890"[:k] for k in range(1, 11)], "١٢٣٤", "²³", "١٢٣٤٥٦٧", "０１２３４", "x12345678y", "3.14159", "2024-10-16", "٣٤٥ ½ Ⅻ",
    # kana/CJK runs, with the punctuation and symbols that lie in the ranges
    "中文テスト・アイ abc123456 !Hello", "ひらがな゠カタカナ゛ー", "東京タワー・スカイツリー", "漢字かな交じり文。句読点、", "カ゚ゞゟ",
    "你好世界，今天天气怎么样？", "日本語123中文", "テスト\nテスト", "中a中", "中 中",
    # ASCII punctuation followed by letters
    "..abc", "don't stop", "foo.bar(baz)", "#include <stdio.h>", "$HOME/.config", "a+b=c", "--verbose -x", "@user", "[link](url)", "'t'é",
    # marks after letters and after spaces
    "é", "naïve café", "á̂b", " ́x", "́́", "क्षत्रिय", "\ń",
    # control and format characters: gaps
    "x\x00\x01 .", "a​b", "a​​.", "\x00\x01\x02", "﻿BOM", "‍‍", "\x1c\x1dz",
    # whitespace and newline runs at the ends of stage pieces
    "a  1", "HELLO world\n\n  end  ", "x   \n\n\t y", "1  中  ", "   ", "\n\n\n", "\r\n\r\n", "end \t", "中 \n", "12 \n ab",
    # specials inside digit runs and CJK runs
    "123" + BOS + "4567", "12" + EOS + "345", "中文" + USER + "テスト", BOS + USER + "hi" + ASSISTANT + "42" + EOS, BOS, EOS + EOS,
    "1" * 300, "中" * 200, "a" * 300, " " * 300, "x" + "́" * 100,
]


def corpus(n, seed):
    words = ("the quick brown fox jumps over lazy dog cache aware router prefix tree worker load token hello world "
             "naïve café déjà Ångström 你好 世界 调度 東京 カタカナ ひらがな テスト・ケース 한국어 12345 2024 3.14159 don't I'll "
             "x=y+1 foo_bar() {\"key\": [1, 2, 3]} https://example.com/a?b=c&d=e \t tab\n newline\r\n crlf   spaces "
             "👋🌍 ＡＢＣ ١٢٣٤ ²³ 's ..abc !Hello #tag @me ~/.bashrc ʼn ệ").split(" ")
    r = random.Random(seed)
    return [" ".join(r.choice(words) for _ in range(r.randrange(1, 40))) for _ in range(n)]


def pre_tokenizer():
    return pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(p), behavior="isolated", invert=False) for p in DEEPSEEK_SPLIT_PATTERNS] +
                                   [pre_tokenizers.ByteLevel(add_prefix_space=False, trim_offsets=True, use_regex=False)])


def build_tokenizer(extra):
    tok = Tokenizer(models.BPE())
    tok.normalizer = normalizers.Sequence([])
    tok.pre_tokenizer = pre_tokenizer()
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=3000, special_tokens=[], initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False)
    tok.train_from_iterator(corpus(4000, 7) + extra, trainer)
    tok.add_special_tokens([AddedToken(s, special=True, normalized=False) for s in SPECIALS])
    return tok


def main():
    tok = build_tokenizer(EDGES)
    open(os.path.join(HERE, FIXTURE), "w").write(tok.to_str(pretty=False))
    saved = json.load(open(os.path.join(HERE, FIXTURE)))
    assert saved["normalizer"] == {"type": "Sequence", "normalizers": []}
    assert [s["pattern"]["Regex"] for s in saved["pre_tokenizer"]["pretokenizers"][:3]] == list(DEEPSEEK_SPLIT_PATTERNS)
    texts = corpus(30, 11) + EDGES
    ids = [e.ids for e in tok.encode_batch(texts, add_special_tokens=False)]
    json.dump({"generator": f"tokenizers {tokenizers.__version__}", "fixture": FIXTURE,
               "cases": [{"text": t, "ids": i} for t, i in zip(texts, ids)]},
              open(os.path.join(HERE, "deepseek_vectors.json"), "w"), ensure_ascii=False)
    print("deepseek texts", len(texts), "vocab", tok.get_vocab_size(), "tokens", sum(len(x) for x in ids))


if __name__ == "__main__":
    main()
