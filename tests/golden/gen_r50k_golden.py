"""Generates the golden fixtures of the GPT-2 (r50k) pre-tokenizer.  Run from the repo root:  python tests/golden/gen_r50k_golden.py

Sources of truth, both offline:
  * Python `tiktoken` 0.12 (OpenAI's Rust CoreBPE) with tiktoken's own GPT-2 pattern `r50k_pat_str` (the regex of r50k_base,
    p50k_base and p50k_edit) over the committed synthetic vocabulary synth_vocab.tiktoken and the specials of bpe_vectors.json;
    no real vocabulary file exists offline.
  * The Python bindings of the `tokenizers` crate: a GPT-2-style tokenizer.json (byte-level BPE, pre-tokenizer
    ByteLevel(add_prefix_space=False, use_regex=True) alone, <|endoftext|> added with normalized=True) trained here.
Outputs (committed):  r50k_vectors.json            texts + expected ids for both, and the oracle form of the pattern
                      hf_gpt2_style_tokenizer.json the tokenizer.json fixture
"""
import base64
import json
import os
import random

import tiktoken
from tiktoken_ext.openai_public import r50k_pat_str
from tokenizers import AddedToken, Tokenizer, decoders, models, pre_tokenizers, trainers

HERE = os.path.dirname(os.path.abspath(__file__))
# The same regex as r50k_pat_str without possessive quantifiers (the form `tokenizers`' ByteLevel uses); oracle/bpe_ref.CoreBPE
# takes it as its `pattern`.
ORACLE_PATTERN = r"'s|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+"
HF_FIXTURE = "hf_gpt2_style_tokenizer.json"

# Where r50k differs from cl100k, and window / special-token edges.
EDGES = [
    "'s", "'S", "'t 'T 're 'RE 've 'Ve 'm 'M 'll 'LL 'lL 'd 'D", "'ſ", "x'ſ", "don't I'll we've they're it's I'M HE'D 'tis",
    " 2024", "1234567", "12345678901234567890 x", "a1b2 3c", " 123 456", "1 12 123 1234 12345",
    "\t1", "　x", "\xa0x", "\t x", "  x", "   1", "\n\n\nx", "\r\n\r\nx", "x\n\n", "a \n b", " \n\n x",
    "!'s", "''s", " 's", "a's", "'''", "' s", "'re'", "a''ll", "!!'ve", "1's", " 'll", "'\n's",
    "x <|endoftext|>", "x  <|endoftext|>", "  <|endoftext|>  ", "\n\n<|endoftext|>\n", "a<|im_start|>'s<|im_end|> 12",
    "<|endoftext|>'s", "'<|endoftext|>s", " <|endoftext|>1", "   ",
    "\x1c\x1d\x1e\x1f x", "\x85x \x85 ", "᠎x​y﻿z", "é é́", "½ Ⅰ ١٢٣ ①", "   　　x",
    "!!!???...,,,;;;:::---___***///", " !!! ??? ...", "http://worker-12:8000/v1/chat/completions?x=1&y=2#frag",
    "你好世界，今天天气怎么样？", "naïve café déjà vu", "emoji \U0001f44b\U0001f30d\U0001f680 mixed", "\U0001d518\U0001d52b 123",
    " " * 300 + "x", "-" * 300, "7" * 300, " " + "!" * 299, "a" * 300 + " " + "b" * 300, "\n" * 300 + "y",
]


def hf_corpus(n, seed):
    words = ("the quick brown fox jumps over lazy dog cache aware router prefix radix tree worker tenant load balance token hello world "
             "naïve café crème brûlée 你好 世界 调度 été ça Straße größer 12345 2024 3.14159 don't I'll we've they're it's x=y+1 foo_bar() "
             "{\"key\": [1, 2, 3]} https://example.com/a?b=c&d=e \t tab\n newline\r\n crlf   spaces   👋🌍 emoji ＡＢＣ ١٢٣ 's 'LL !'s").split(" ")
    r = random.Random(seed)
    return [" ".join(r.choice(words) for _ in range(r.randrange(1, 40))) for _ in range(n)]


def build_hf(extra):
    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=True)
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=2500, special_tokens=[], initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False)
    tok.train_from_iterator(hf_corpus(4000, 7) + extra, trainer)
    tok.add_special_tokens([AddedToken("<|endoftext|>", special=True, normalized=True)])
    return tok


def main():
    bpe = json.load(open(os.path.join(HERE, "bpe_vectors.json")))
    specials = bpe["specials"]
    ranks = {}
    for line in open(os.path.join(HERE, "synth_vocab.tiktoken")).read().splitlines():
        if line:
            t, r = line.split()
            ranks[base64.b64decode(t)] = int(r)
    enc = tiktoken.Encoding("synth_r50k", pat_str=r50k_pat_str, mergeable_ranks=ranks, special_tokens=specials)
    texts = [c["text"] for c in bpe["cases"]][::4] + EDGES   # every 4th cl100k golden text: the stress set, code, chat turns, specials
    cases = [{"text": t, "ids": enc.encode(t, allowed_special="all")} for t in texts]

    tok = build_hf([c["text"] for c in bpe["cases"]])   # the golden texts widen the corpus so that the vocabulary fills up
    open(os.path.join(HERE, HF_FIXTURE), "w").write(tok.to_str(pretty=False))
    saved = json.load(open(os.path.join(HERE, HF_FIXTURE)))
    assert [a["normalized"] for a in saved["added_tokens"]] == [True]
    hf_texts = hf_corpus(60, 11) + EDGES + ["<|endoftext|>hello world<|endoftext|>", "a<|endoftext|>'s", "<|endoftext|<|endoftext|>>"]
    hf_ids = [e.ids for e in tok.encode_batch(hf_texts, add_special_tokens=False)]

    json.dump({"generator": f"tiktoken {tiktoken.__version__} (pat_str = r50k_pat_str); tokenizers (ByteLevel use_regex=True)",
               "pattern": ORACLE_PATTERN, "tiktoken_pattern": r50k_pat_str, "specials": specials, "cases": cases,
               "hf": {"fixture": HF_FIXTURE, "texts": hf_texts, "ids": hf_ids}},
              open(os.path.join(HERE, "r50k_vectors.json"), "w"), ensure_ascii=True)
    print("tiktoken cases", len(cases), "tokens", sum(len(c["ids"]) for c in cases), "| hf texts", len(hf_texts),
          "vocab", tok.get_vocab_size(), "tokens", sum(len(x) for x in hf_ids))


if __name__ == "__main__":
    main()
