"""CPU only: the GPT-2 (r50k) pattern with the BPE oracle (oracle/bpe_ref.py, which takes its pattern as an argument) against the
golden vectors that tests/golden/gen_r50k_golden.py recorded from tiktoken's `r50k_pat_str`, and, when the packages import, its
pieces against live tiktoken and the `tokenizers` ByteLevel(use_regex=True) pre-tokenizer on random text."""
import json
import os
import random

import pytest

from oracle import bpe_ref

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ALPHABET = ("abcdefghij XYZ 0123456789 sdmtlvrSDMTLVRe '''\n\n\r\t\t  .,!?-_()" + "\x1c\x1d\x1e\x1f\x85\xa0᠎​　﻿́"
            + "½Ⅰ١٢éß你好\U0001f44b")


def _load():
    g = json.load(open(os.path.join(GOLD, "r50k_vectors.json")))
    return g, bpe_ref.load_tiktoken_bpe(os.path.join(GOLD, "synth_vocab.tiktoken"))


def _random_texts(seed, n, maxlen):
    rng = random.Random(seed)
    return ["".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, maxlen))) for _ in range(n)]


def test_golden_pattern_is_the_gpt2_pattern():
    g, _ = _load()
    assert g["pattern"] == r"'s|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+"
    tiktoken_ext = pytest.importorskip("tiktoken_ext.openai_public")
    assert g["tiktoken_pattern"] == tiktoken_ext.r50k_pat_str


def test_oracle_matches_r50k_golden_vectors():
    g, ranks = _load()
    enc = bpe_ref.CoreBPE(ranks, g["specials"], pattern=g["pattern"])
    assert len(g["cases"]) > 150
    for c in g["cases"]:
        assert enc.encode_with_special_tokens(c["text"]) == c["ids"], repr(c["text"][:80])


def test_oracle_pieces_equal_live_tiktoken_pieces():
    tiktoken = pytest.importorskip("tiktoken")
    g, ranks = _load()
    live = tiktoken.Encoding("synth_r50k", pat_str=g["tiktoken_pattern"], mergeable_ranks=ranks, special_tokens={})
    enc = bpe_ref.CoreBPE(ranks, {}, pattern=g["pattern"])
    for t in _random_texts(51, 3000, 80):
        ids = live.encode_ordinary(t)
        assert enc.encode_ordinary(t) == ids, repr(t)
    # piece level: tiktoken's regex directly (the `regex` module accepts its possessive form)
    import regex
    rx = regex.compile(g["tiktoken_pattern"])
    for t in _random_texts(52, 3000, 80):
        assert enc.pieces(t) == rx.findall(t), repr(t)


def test_oracle_pieces_equal_tokenizers_byte_level_pieces():
    tokenizers = pytest.importorskip("tokenizers")
    g, ranks = _load()
    enc = bpe_ref.CoreBPE(ranks, {}, pattern=g["pattern"])
    pre = tokenizers.pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=True)
    from smg_b200.policy import _byte_level_decoder
    dec = _byte_level_decoder()
    for t in _random_texts(53, 3000, 80):
        got = [bytes(dec[c] for c in p).decode() for p, _ in pre.pre_tokenize_str(t)]
        assert enc.pieces(t) == got, repr(t)
