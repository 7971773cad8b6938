"""CPU only: loading Qwen2-family tokenizer.json files (NFC normalizer, the single-digit Split) on a host-mirror policy (device_id = -1),
the shapes that stay refused, and unknown enum values at the ABI.  Encoding needs the GPU (tests/test_gpu_tokenizer_qwen2.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from smg_b200 import SmgxError, _lib
from smg_b200.policy import LLAMA3_SPLIT_PATTERN, QWEN2_SPLIT_PATTERN, CacheAwareConfig, HuggingFaceTokenizer, _Handle

GOLD = os.path.join(os.path.dirname(__file__), "golden")
NFC_SEQ = {"type": "Sequence", "normalizers": [{"type": "NFC"}]}


def _load(tmp_path, j):
    (tmp_path / "t.json").write_text(json.dumps(j))
    return HuggingFaceTokenizer(_Handle(CacheAwareConfig(eviction_interval_secs=0), -1), "unknown", str(tmp_path / "t.json"))


def _file(name, **top):
    j = json.load(open(os.path.join(GOLD, name)))
    j.update(top)
    if name == "hf_gpt2_style_tokenizer.json":
        for a in j["added_tokens"]:
            a["normalized"] = False
    return j


@pytest.mark.parametrize("name,top,growth", [
    ("hf_qwen2_style_tokenizer.json", {}, 3), ("hf_qwen2_style_tokenizer.json", {"normalizer": None}, 1),
    ("hf_qwen2_style_tokenizer.json", {"normalizer": NFC_SEQ}, 3), ("hf_gpt2_style_tokenizer.json", {"normalizer": {"type": "NFC"}}, 3),
    ("hf_gpt2_style_tokenizer.json", {"normalizer": NFC_SEQ}, 3)])
def test_accepted_files_load_and_encode_fails_loudly_without_device(tmp_path, name, top, growth):
    tok = _load(tmp_path, _file(name, **top))
    assert tok.growth == growth
    with pytest.raises(SmgxError):
        tok.encode("héllo 123")


@pytest.mark.parametrize("mutate", [
    *[lambda j, n=n: j.update(normalizer=n) for n in ({"type": "NFKC"}, {"type": "NFD"}, {"type": "Lowercase"}, {"type": "Prepend", "prepend": "▁"},
                                                      {"type": "Sequence", "normalizers": [{"type": "NFC"}, {"type": "Lowercase"}]},
                                                      {"type": "Sequence", "normalizers": []})],
    lambda j: [a.update(normalized=True) for a in j["added_tokens"]],                        # matched on normalized text
    lambda j: j["added_tokens"][0].update(normalized=True),                                  # mixed
    lambda j: j["pre_tokenizer"]["pretokenizers"][0]["pattern"].update(Regex=QWEN2_SPLIT_PATTERN[:-1]),
    lambda j: j["pre_tokenizer"]["pretokenizers"][0]["pattern"].update(Regex=QWEN2_SPLIT_PATTERN.replace(r"\p{N}|", r"\p{N}{1,2}|")),
    lambda j: j["pre_tokenizer"]["pretokenizers"][0]["pattern"].update(Regex=LLAMA3_SPLIT_PATTERN),   # Llama-3 Split with NFC
    lambda j: j["pre_tokenizer"]["pretokenizers"][1].update(add_prefix_space=True),
])
def test_unsupported_configurations_are_refused(tmp_path, mutate):
    j = _file("hf_qwen2_style_tokenizer.json")
    mutate(j)
    with pytest.raises(ValueError):
        _load(tmp_path, j)


def test_abi_refuses_unknown_enum_values():
    h, L = _Handle(CacheAwareConfig(eviction_interval_secs=0), -1), _lib.load()
    blob, offs, ids = np.arange(256, dtype=np.uint8), np.arange(257, dtype=np.uint32), np.arange(256, dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731

    def load(pt, nm):
        err = C.c_char_p()
        st = L.smgx_tokenizer_load_bpe_merges_norm(h.p, b"m", p(blob), p(offs), p(ids), 256, None, 0, 0, None, None, 0, pt, nm, C.byref(err))
        msg = err.value
        if msg is not None:
            L.smgx_free_string(C.cast(err, C.c_void_p))
        return st, msg
    for pt in (_lib.PRETOK_CL100K, _lib.PRETOK_R50K, _lib.PRETOK_QWEN2):
        for nm in (_lib.NORMALIZER_NONE, _lib.NORMALIZER_NFC):
            assert load(pt, nm) == (_lib.SUCCESS, None)
    for pt, nm, word in ((3, 0, b"pretokenizer"), (-1, 0, b"pretokenizer"), (0, 2, b"normalizer"), (2, -1, b"normalizer")):
        st, msg = load(pt, nm)
        assert st == _lib.INVALID_ARGUMENT and word in msg, (pt, nm, msg)
    for pt, want in ((_lib.PRETOK_QWEN2, _lib.SUCCESS), (3, _lib.INVALID_ARGUMENT)):   # the tiktoken loaders take the Qwen2 pattern too
        assert L.smgx_tokenizer_load_tiktoken_ex(h.p, b"m", p(blob), p(offs), p(ids), 256, None, None, 0, pt, None) == want
