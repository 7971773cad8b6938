"""CPU only: the SentencePiece-style BPE stages (metaspace.cuh: ▁ normalization, segmenter, character-level symbolizer; bpe.cuh
merge_symbols), built for the host by tests/cpp/metaspace.mk, against live `tokenizers` on the Llama-2-style fixture in every accepted
shape.  Each text is encoded twice: with every piece merged on its own (what the GPU does) and with every stretch merged as one word (what
`tokenizers` does); both must give the ids `tokenizers` gives."""
import json
import os
import random
import struct
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
GOLD = os.path.join(ROOT, "tests", "golden")
FIXTURE = os.path.join(GOLD, "hf_llama2_style_tokenizer.json")
SPECIALS = ["<unk>", "<s>", "</s>", "<|user|>", "<|assistant|>"]
# spaces, ▁ written out, specials, byte-fallback characters (emoji, tab, newline, rare CJK), vocabulary characters, combining marks
AWKWARD = [" ", " ", "  ", "▁", "▁▁", "\t", "\n", "\r\n", "a", "b", "the", "he", "é", "é", "中", "文", "龍", "😀", "👋🌍", "‍", "̣",
           "<0x41>", "<", "s>"] + SPECIALS
# (prepend argument of the harness, split) per variant; the harness's prepend codes follow metaspace.cuh's MS_PREPEND_*
VARIANTS = {"legacy": (3, 0), "metaspace-first-nosplit": (1, 0), "metaspace-always-nosplit": (2, 0), "metaspace-first-split": (1, 1),
            "metaspace-never-nosplit": (0, 0), "metaspace-always-split": (2, 1), "metaspace-never-split": (0, 1)}


def variant_json(name):
    j = json.load(open(FIXTURE))
    if name != "legacy":
        _, scheme, split = name.split("-")
        j["normalizer"] = None
        j["pre_tokenizer"] = {"type": "Metaspace", "replacement": "▁", "prepend_scheme": scheme, "split": split == "split"}
    return j


def _model_blob(j):
    u = lambda *xs: struct.pack(f"<{len(xs)}I", *xs)   # noqa: E731
    vocab = j["model"]["vocab"]
    out = [u(len(vocab))] + [u(i, len(s.encode())) + s.encode() for s, i in vocab.items()]
    out += [u(len(j["model"]["merges"]))] + [u(vocab[a], vocab[b]) for a, b in j["model"]["merges"]]
    added = j["added_tokens"]
    out += [u(len(added))] + [u(a["id"], len(a["content"].encode())) + a["content"].encode() for a in added]
    return b"".join(out)


def _run(name, texts):
    subprocess.check_call(["make", "-s", "-C", CPP, "-f", "metaspace.mk", "test_metaspace_host"])
    prepend, split = VARIANTS[name]
    blob = _model_blob(variant_json(name)) + b"".join(struct.pack("<I", len(b)) + b for b in (t.encode() for t in texts))
    lines = subprocess.run([os.path.join(CPP, "test_metaspace_host"), str(prepend), str(split)], input=blob, capture_output=True,
                           timeout=600, check=True).stdout.decode().splitlines()
    assert len(lines) == 2 * len(texts)
    nums = lambda ln: [int(x) for x in ln.split()[1:]]   # noqa: E731
    return [(nums(lines[2 * k]), nums(lines[2 * k + 1])) for k in range(len(texts))]


def _texts(seed, n):
    rng = random.Random(seed)
    texts = [c["text"] for c in json.load(open(os.path.join(GOLD, "llama2_vectors.json")))["cases"]]
    return texts + ["".join(rng.choice(AWKWARD) for _ in range(rng.randint(0, 40))) for _ in range(n)]


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_pieces_and_whole_stretches_equal_live_tokenizers(name):
    """20 000 random strings per variant: the GPU's independent pieces, and whole stretches, give what `tokenizers` gives."""
    tk = pytest.importorskip("tokenizers").Tokenizer.from_str(json.dumps(variant_json(name)))
    texts = _texts(len(name), 20000)
    want = [e.ids for e in tk.encode_batch(texts, add_special_tokens=False)]
    split, n_cut = VARIANTS[name][1], 0
    for t, w, (pieces, whole) in zip(texts, want, _run(name, texts)):
        assert pieces == w, (name, repr(t))
        if not split:   # with split the cut before every ▁ is part of the semantics: there is no whole-stretch word
            assert whole == w, (name, repr(t))
        n_cut += " " in t or "▁" in t
    assert n_cut > 10000


def test_goldens_of_the_committed_variants():
    g = json.load(open(os.path.join(GOLD, "llama2_vectors.json")))
    texts = [c["text"] for c in g["cases"]]
    for name, ids in g["variants"].items():
        assert [p for p, _ in _run(name, texts)] == ids, name
