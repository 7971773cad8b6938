"""CPU only: the GPT-2 (r50k) pre-tokenizer of smg_b200/csrc/bpe.cuh (next_piece_r50k + the r50k anchor rule), built for the host by
tests/cpp/splitter.mk, against the regex.  On every text: the serial split equals the regex's pieces, every anchor is a piece start,
and the anchored split the GPU kernel does equals the serial one.  A wrong hand-compiled alternative or anchor rule fails here
before any GPU run."""
import json
import os
import random
import struct
import subprocess

import regex

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
GOLD = os.path.join(ROOT, "tests", "golden")
# ASCII and the characters where classes are easy to get wrong: \x1c-\x1f and U+0085 (whitespace in some tables, not in others),
# U+00A0, U+180E, U+200B, U+3000, U+FEFF, a combining mark, ½, Ⅰ, Arabic-Indic digits, CJK and an astral emoji.
AWKWARD = ("abcdefghij XYZ 0123456789 sdmtlvrSDMTLVRe '''\n\n\r\t\t  .,!?-_()<|>" + "\x1c\x1d\x1e\x1f\x85\xa0᠎​　﻿́"
           + "½Ⅰ١٢éß你好\U0001f44b")


def _pattern():
    return json.load(open(os.path.join(GOLD, "r50k_vectors.json")))["pattern"]


def _split(texts):
    subprocess.check_call(["make", "-s", "-C", CPP, "-f", "splitter.mk", "test_r50k_splitter"])
    blob = b"".join(struct.pack("<I", len(b)) + b for b in (t.encode() for t in texts))
    out = subprocess.run([os.path.join(CPP, "test_r50k_splitter")], input=blob, capture_output=True, timeout=300, check=True).stdout
    lines = out.decode().splitlines()
    assert len(lines) == 3 * len(texts)
    nums = lambda ln: [int(x) for x in ln.split()[1:]]   # noqa: E731
    return [(nums(lines[3 * k]), nums(lines[3 * k + 1]), nums(lines[3 * k + 2])) for k in range(len(texts))]


def _regex_starts(rx, text):
    starts, pos = [], 0
    for m in rx.finditer(text):
        assert m.start() == pos     # the pattern matches every character, so pieces tile the text
        starts.append(len(text[:pos].encode()))
        pos = m.end()
    assert pos == len(text)
    return starts


def _texts():
    rng = random.Random(50)
    texts = [c["text"] for c in json.load(open(os.path.join(GOLD, "r50k_vectors.json")))["cases"]]
    texts += ["".join(rng.choice(AWKWARD) for _ in range(rng.randint(0, 60))) for _ in range(20000)]
    return [t for t in texts if "<|" not in t]   # specials are cut out before the regex; the GPU tests cover them


def test_serial_split_equals_regex_and_anchors_are_piece_starts():
    rx = regex.compile(_pattern())
    texts = _texts()
    n_anchor = n_start = 0
    for t, (starts, anchors, seg) in zip(texts, _split(texts)):
        want = _regex_starts(rx, t)
        assert starts == want, (repr(t), starts, want)
        assert set(anchors) <= set(starts), (repr(t), sorted(set(anchors) - set(starts)))
        assert seg == starts, repr(t)
        n_anchor += len(anchors)
        n_start += len(starts)
    assert n_anchor > n_start // 2   # the rule must also be useful: most piece starts are anchors


def test_edges_of_the_issue_list():
    """The cases where r50k differs from cl100k, spelled out."""
    cases = {"'s": ["'s"], "'S": ["'", "S"], "'LL": ["'", "LL"], "'ſ": ["'", "ſ"], " 2024": [" 2024"], "1234567": ["1234567"],
             "\t1": ["\t", "1"], "　x": ["　", "x"], "\xa0x": ["\xa0", "x"], "\n\n\nx": ["\n\n", "\n", "x"],
             "!'s": ["!'", "s"], "''s": ["''", "s"], " 's": [" '", "s"], "a's": ["a", "'s"], " 123": [" 123"]}
    texts = list(cases)
    for t, (starts, anchors, _) in zip(texts, _split(texts)):
        b = t.encode()
        pieces = [b[s:e].decode() for s, e in zip(starts, starts[1:] + [len(b)])]
        assert pieces == cases[t], repr(t)
        assert set(anchors) <= set(starts)
