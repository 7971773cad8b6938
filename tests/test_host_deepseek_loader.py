"""CPU only: loading DeepSeek-V3-family tokenizer.json files (the chain of three Splits) on a host-mirror policy (device_id = -1), every
mutation of the shape that stays refused, the `normalized` marks of the added tokens, and SMGX_PRETOK_DEEPSEEK at the ABI.  Encoding needs
the GPU (tests/test_gpu_tokenizer_deepseek.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from smg_b200 import SmgxError, _lib
from smg_b200.policy import DEEPSEEK_SPLIT_PATTERNS, CacheAwareConfig, HuggingFaceTokenizer, _Handle

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIXTURE = os.path.join(GOLD, "hf_deepseek_v3_style_tokenizer.json")


def _load(tmp_path, j):
    (tmp_path / "t.json").write_text(json.dumps(j))
    return HuggingFaceTokenizer(_Handle(CacheAwareConfig(eviction_interval_secs=0), -1), "unknown", str(tmp_path / "t.json"))


def _steps(j):
    return j["pre_tokenizer"]["pretokenizers"]


def _marks(*values):
    def mutate(j):
        for a, v in zip(j["added_tokens"], values):
            a["normalized"] = v
    return mutate


@pytest.mark.parametrize("mutate", [
    lambda j: None,
    lambda j: j.update(normalizer=None),
    lambda j: _steps(j)[3].update(trim_offsets=False),
    lambda j: j["model"].update(ignore_merges=True),
    lambda j: j["model"].update(ignore_merges=False),
    _marks(True, True, True, True),
    _marks(True, False, True, False),   # mixed: no two of these strings can overlap in a text
])
def test_accepted_files_load_and_encode_fails_loudly_without_device(tmp_path, mutate):
    j = json.load(open(FIXTURE))
    mutate(j)
    tok = _load(tmp_path, j)
    assert tok.growth == 1
    with pytest.raises(SmgxError):
        tok.encode("中文テスト 123456")


def _pattern(k, regex):
    return lambda j: _steps(j)[k].update(pattern={"Regex": regex})


@pytest.mark.parametrize("mutate", [
    _pattern(0, "\\p{N}{1,2}"), _pattern(0, "\\p{N}"),
    _pattern(1, "[一-龥぀-ゟ]+"), _pattern(1, DEEPSEEK_SPLIT_PATTERNS[1][:-1]),
    _pattern(2, DEEPSEEK_SPLIT_PATTERNS[2][:-1]), _pattern(2, DEEPSEEK_SPLIT_PATTERNS[2].replace("[A-Za-z]+", "[A-Za-z]*")),
    _pattern(2, DEEPSEEK_SPLIT_PATTERNS[2].replace("\r\n", "\\r\\n")),
    lambda j: _steps(j).__setitem__(slice(0, 2), _steps(j)[1::-1]),            # Splits reordered
    lambda j: _steps(j).__setitem__(slice(1, 3), _steps(j)[2:0:-1]),
    lambda j: _steps(j).pop(1),                                                 # one dropped
    lambda j: _steps(j).pop(0),
    lambda j: _steps(j).insert(3, dict(_steps(j)[2])),                          # one extra
    lambda j: _steps(j).pop(3),                                                 # no ByteLevel
    *[lambda j, k=k, b=b: _steps(j)[k].update(behavior=b) for k in range(3) for b in ("Removed", "MergedWithPrevious")],
    *[lambda j, k=k: _steps(j)[k].update(invert=True) for k in range(3)],
    lambda j: _steps(j)[3].update(use_regex=True),
    lambda j: _steps(j)[3].update(add_prefix_space=True),
    lambda j: _steps(j)[3].pop("use_regex"),                                    # the crate's default is true
    *[lambda j, n=n: j.update(normalizer=n) for n in ({"type": "NFC"}, {"type": "Sequence", "normalizers": [{"type": "NFC"}]},
                                                      {"type": "Lowercase"}, {"type": "Sequence", "normalizers": [{"type": "NFKC"}]})],
    lambda j: j["model"].update(byte_fallback=True),
    lambda j: j["added_tokens"][0].update(lstrip=True),
])
def test_mutated_shapes_are_refused(tmp_path, mutate):
    j = json.load(open(FIXTURE))
    mutate(j)
    with pytest.raises(ValueError):
        _load(tmp_path, j)


def test_mixed_marks_on_overlapping_added_tokens_are_refused(tmp_path):
    """`tokenizers` cuts the normalized = false tokens first: with "<｜User｜>x" normalized and "x<｜A" not, the marks decide the split."""
    j = json.load(open(FIXTURE))
    n = max(a["id"] for a in j["added_tokens"]) + 1
    j["added_tokens"] += [dict(j["added_tokens"][0], id=n, content="<｜U", normalized=True),
                          dict(j["added_tokens"][0], id=n + 1, content="U｜>x<", normalized=False)]
    with pytest.raises(ValueError, match="overlap"):
        _load(tmp_path, j)


def test_deepseek_shape_does_not_open_other_shapes(tmp_path):
    """The empty-Sequence normalizer and mixed marks stay refused on every other shape."""
    q = json.load(open(os.path.join(GOLD, "hf_qwen2_style_tokenizer.json")))
    q["normalizer"] = {"type": "Sequence", "normalizers": []}
    with pytest.raises(ValueError):
        _load(tmp_path, q)
    q = json.load(open(os.path.join(GOLD, "hf_qwen2_style_tokenizer.json")))
    q["normalizer"] = None
    q["added_tokens"][0]["normalized"] = True
    with pytest.raises(ValueError):
        _load(tmp_path, q)


def test_abi_accepts_4_and_refuses_3_and_7():
    h, L = _Handle(CacheAwareConfig(eviction_interval_secs=0), -1), _lib.load()
    blob, offs, ids = np.arange(256, dtype=np.uint8), np.arange(257, dtype=np.uint32), np.arange(256, dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert _lib.PRETOK_DEEPSEEK == 4
    for pt, want in ((4, _lib.SUCCESS), (3, _lib.INVALID_ARGUMENT), (7, _lib.INVALID_ARGUMENT)):
        assert L.smgx_tokenizer_load_bpe_merges_norm(h.p, b"m", p(blob), p(offs), p(ids), 256, None, 0, 0, None, None, 0, pt,
                                                     _lib.NORMALIZER_NONE, None) == want, pt
        assert L.smgx_tokenizer_load_bpe_merges_ex(h.p, b"m", p(blob), p(offs), p(ids), 256, None, 0, 0, None, None, 0, pt, None) == want, pt
        assert L.smgx_tokenizer_load_tiktoken_ex(h.p, b"m", p(blob), p(offs), p(ids), 256, None, None, 0, pt, None) == want, pt
