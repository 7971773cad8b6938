"""CPU only: the Qwen2 pre-tokenizer (bpe.cuh) and the NFC normalizer (nfc.cuh), built for the host by tests/cpp/qwen2.mk, against the
regex of the Qwen2 Split and against live `tokenizers` NFC (the crate behind HuggingFaceTokenizer::encode)."""
import json
import os
import random
import struct
import subprocess
import sys
import unicodedata

import pytest
import regex

from smg_b200.policy import QWEN2_SPLIT_PATTERN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
GOLD = os.path.join(ROOT, "tests", "golden")
AWKWARD = ("abcdefghij XYZ 0123456789 sdmtlvrSDMTLVRe '''\n\n\r\t\t  .,!?-_()<|>\x1c\x1d\x1e\x1f\x85\xa0᠎​　﻿́"
           "½Ⅰ١٢éßſ你\U0001f44b²³०")


def _run(mode, texts):
    subprocess.check_call(["make", "-s", "-C", CPP, "-f", "qwen2.mk", "test_qwen2_host"])
    blob = b"".join(struct.pack("<I", len(b)) + b for b in (t.encode() for t in texts))
    return subprocess.run([os.path.join(CPP, "test_qwen2_host"), mode], input=blob, capture_output=True, timeout=600, check=True).stdout


def _split(texts):
    lines = _run("split", texts).decode().splitlines()
    assert len(lines) == 3 * len(texts)
    nums = lambda ln: [int(x) for x in ln.split()[1:]]   # noqa: E731
    return [(nums(lines[3 * k]), nums(lines[3 * k + 1]), nums(lines[3 * k + 2])) for k in range(len(texts))]


def test_split_equals_regex_and_anchors_are_piece_starts():
    """The serial split equals the regex's pieces, every anchor starts a piece, the anchored split equals the serial one."""
    rx = regex.compile(QWEN2_SPLIT_PATTERN)
    rng = random.Random(2)
    texts = [c["text"] for c in json.load(open(os.path.join(GOLD, "qwen2_vectors.json")))["cases"]]
    texts += [c["text"] for c in json.load(open(os.path.join(GOLD, "r50k_vectors.json")))["cases"]]
    texts += ["".join(rng.choice(AWKWARD) for _ in range(rng.randint(0, 60))) for _ in range(20000)]
    texts = [t for t in texts if "<|" not in t] + ["12345", "a1b", " 42x", "I'M 7", "\n\n1"]   # specials: cut before the regex
    n_anchor = n_start = 0
    for t, (starts, anchors, seg) in zip(texts, _split(texts)):
        want = [len(t[:m.start()].encode()) for m in rx.finditer(t)]
        assert starts == want, repr(t)
        assert set(anchors) <= set(starts) and seg == starts, repr(t)
        n_anchor, n_start = n_anchor + len(anchors), n_start + len(starts)
    assert n_anchor > n_start // 2


def _check_nfc(texts):
    tk = pytest.importorskip("tokenizers.normalizers").NFC().normalize_str
    out, pos, got = _run("nfc", texts), 0, []
    while pos < len(out):
        (n,) = struct.unpack_from("<I", out, pos)
        got.append(out[pos + 4:pos + 4 + n].decode())
        pos += 4 + n
    assert len(got) == 2 * len(texts)
    for k, t in enumerate(texts):
        assert got[2 * k] == got[2 * k + 1] == tk(t), [hex(ord(c)) for c in t[:40]]


def test_nfc_every_code_point_and_every_composite():
    cps = [cp for cp in range(0x110000) if not 0xD800 <= cp <= 0xDFFF]
    nfd = [unicodedata.normalize("NFD", chr(cp)) for cp in cps]
    texts = ["".join(chr(cp) for cp in cps[k:k + 64]) for k in range(0, len(cps), 64)]
    texts += [chr(cp) for cp, d in zip(cps, nfd) if unicodedata.combining(chr(cp)) or d != chr(cp)] + [d for cp, d in zip(cps, nfd) if d != chr(cp)]
    _check_nfc(texts)


def test_nfc_random_sequences_and_long_runs():
    """200 000 seeded sequences of marks (the 108 that `tokenizers` gives class 0 included), starters, composites and jamo; runs of 3000
    mixed-class marks, far past the 32-entry short path."""
    pytest.importorskip("tokenizers")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_nfc_tables as gen
    sys.path.pop(0)
    ccc, dec, comp, zeroed, _, _ = gen.build()
    rng = random.Random(7)
    pools = [sorted(ccc) + zeroed, sorted({a for a, _ in comp}) + [0x41, 0x4E00, 0x20], sorted({b for _, b in comp}), sorted(comp.values()),
             list(range(0x1100, 0x1113)) + sorted(gen.SECOND_JAMO) + [0xAC00, 0xAC01, 0xD7A3]]
    texts = ["".join(chr(rng.choice(rng.choice(pools))) for _ in range(rng.randint(1, 12))) for _ in range(200000)]
    marks = [chr(cp) for cp in pools[0]]
    texts += [b + "".join(rng.choice(marks) for _ in range(3000)) for b in ("a", "e", "ᄀ", "가", "一", "େ", "")]
    texts += ["ᄀ" + "ᅡ" * 3000, "\U0001d160" * 1000]
    _check_nfc(texts)


def test_committed_tables_match_the_generator():
    pytest.importorskip("tokenizers")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "gen_nfc_tables.py"), "--check"])
