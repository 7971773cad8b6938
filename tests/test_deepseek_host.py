"""CPU only: the DeepSeek pre-tokenizer (bpe.cuh, next_piece_deepseek and its anchor rule) on the deepseek_tables.h classes, built for the
host by tests/cpp/deepseek.mk, against live `tokenizers` (the crate behind HuggingFaceTokenizer::encode): the split of the Sequence of
three Splits, and the class of every code point."""
import json
import os
import random
import struct
import subprocess
import sys

import pytest

from smg_b200.policy import DEEPSEEK_SPLIT_PATTERNS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
GOLD = os.path.join(ROOT, "tests", "golden")
# digits of several scripts, kana/CJK with the punctuation and symbols inside the ranges (U+30A0 Pd, U+30FB Po, U+309B Sk), the voicing
# marks U+3099/U+309A, unassigned U+3097, a CJK ideograph past U+9FA5, ASCII punctuation before letters, marks, format and control
# characters (gaps), and whitespace of every kind
AWKWARD = ("abcXYZ é 0123456789 ١٢٣²³½Ⅳ０ 中文テスト・゠゛ゞ゚゗鿿가 .,!?'\"-_()<|>$+^`~@#\\/{}「」、。 "
           "́̀ि \x00\x01\x1c​‍﻿\U000e0001 \n\n\r\t\t\x0b\x0c\x85\xa0 　 \U0001f44b")


def _run(mode, blob=b""):
    subprocess.check_call(["make", "-s", "-C", CPP, "-f", "deepseek.mk", "test_deepseek_host"])
    return subprocess.run([os.path.join(CPP, "test_deepseek_host"), mode], input=blob, capture_output=True, timeout=600, check=True).stdout


def _split(texts):
    blob = b"".join(struct.pack("<I", len(b)) + b for b in (t.encode() for t in texts))
    lines = _run("split", blob).decode().splitlines()
    assert len(lines) == 3 * len(texts)
    nums = lambda ln: [int(x) for x in ln.split()[1:]]   # noqa: E731
    return [(nums(lines[3 * k]), nums(lines[3 * k + 1]), nums(lines[3 * k + 2])) for k in range(len(texts))]


def _reference():
    """The pre_tokenizer of the DeepSeek tokenizer.json without its ByteLevel step."""
    tk = pytest.importorskip("tokenizers")
    pt = tk.pre_tokenizers
    return pt.Sequence([pt.Split(tk.Regex(p), behavior="isolated", invert=False) for p in DEEPSEEK_SPLIT_PATTERNS])


def test_split_equals_tokenizers_and_anchors_are_piece_starts():
    """The serial split equals `tokenizers`' pieces, every anchor starts a piece, the anchored split equals the serial one."""
    ref = _reference()
    rng = random.Random(4)
    texts = [c["text"] for c in json.load(open(os.path.join(GOLD, "deepseek_vectors.json")))["cases"]]
    texts += ["".join(rng.choice(AWKWARD) for _ in range(rng.randint(0, 60))) for _ in range(20000)]
    texts += ["".join(rng.choice("0١²中テ・a. \n") for _ in range(rng.randint(0, 40))) for _ in range(5000)]
    texts = [t for t in texts if "<｜" not in t]   # specials are cut before the pre-tokenizer
    texts += ["a  1", "x\x00\x01 .", "..abc", "don't stop", "中文テスト・アイ abc123456 !Hello", "HELLO world\n\n  end  ", "a​b",
              "12345678", "1" * 1000]
    n_anchor = n_start = 0
    for t, (starts, anchors, seg) in zip(texts, _split(texts)):
        want = [len(t[:a].encode()) for _, (a, _) in ref.pre_tokenize_str(t)]   # offsets count code points
        assert starts == want, repr(t)
        assert set(anchors) <= set(starts) and seg == starts, repr(t)
        n_anchor, n_start = n_anchor + len(anchors), n_start + len(starts)
    assert n_anchor > n_start // 2


def test_every_code_point_has_the_tokenizers_class():
    """ds_class() — the ASCII rules it hard-codes and the committed table — equals live `tokenizers` on every code point."""
    pytest.importorskip("tokenizers")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_deepseek_tables as gen
    sys.path.pop(0)
    got = _run("classes")
    assert len(got) == 0x110000
    want = gen.build()
    bad = [cp for cp, c in want.items() if got[cp] != c]
    assert not bad, [(hex(cp), got[cp], want[cp]) for cp in bad[:20]]


def test_committed_table_matches_the_generator():
    pytest.importorskip("tokenizers")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "gen_deepseek_tables.py"), "--check"])
