"""CPU only: loading GPT-2 (r50k) tokenizers on a host-mirror policy (device_id = -1): the tiktoken encodings that use the pattern, the
GPT-2-style tokenizer.json, the shapes that stay refused, and the pretokenizer argument of the _ex loaders.  Encoding needs the GPU
(tests/test_gpu_tokenizer_r50k.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from smg_b200 import SmgxError, _lib
from smg_b200.policy import CacheAwareConfig, HuggingFaceTokenizer, TiktokenTokenizer, _Handle

GOLD = os.path.join(os.path.dirname(__file__), "golden")
VOCAB = os.path.join(GOLD, "synth_vocab.tiktoken")
GPT2 = os.path.join(GOLD, "hf_gpt2_style_tokenizer.json")


def _host():
    return _Handle(CacheAwareConfig(eviction_interval_secs=0), -1)


def _write(tmp_path, j, name="tokenizer.json"):
    p = tmp_path / name
    p.write_text(json.dumps(j))
    return str(p)


@pytest.mark.parametrize("encoding", ["cl100k_base", "r50k_base", "p50k_base", "p50k_edit"])
def test_tiktoken_encodings_load_and_encode_fails_loudly_without_device(encoding):
    tok = TiktokenTokenizer(_host(), "unknown", VOCAB, {"<|endoftext|>": 3000}, encoding=encoding)
    with pytest.raises(SmgxError):
        tok.encode("hello 's 2024")


@pytest.mark.parametrize("encoding", ["o200k_base", "gpt2", "R50K_BASE", ""])
def test_unknown_tiktoken_encoding_is_refused(encoding):
    with pytest.raises(ValueError):
        TiktokenTokenizer(_host(), "unknown", VOCAB, None, encoding=encoding)


def test_gpt2_style_files_load_and_encode_fails_loudly_without_device(tmp_path):
    """The fixture; its ByteLevel as a one-element Sequence; a Llama-3-style file with every added token marked normalized."""
    seq = json.load(open(GPT2))
    seq["pre_tokenizer"] = {"type": "Sequence", "pretokenizers": [seq["pre_tokenizer"]]}
    llama = json.load(open(os.path.join(GOLD, "hf_llama3_style_tokenizer.json")))
    for a in llama["added_tokens"]:
        a["normalized"] = True
    for path in (GPT2, _write(tmp_path, seq, "seq.json"), _write(tmp_path, llama, "llama.json")):
        tok = HuggingFaceTokenizer(_host(), "unknown", path)
        with pytest.raises(SmgxError):
            tok.encode("hello")


@pytest.mark.parametrize("mutate", [
    lambda j: j["pre_tokenizer"].update(add_prefix_space=True),                                      # RoBERTa
    lambda j: j["pre_tokenizer"].update(use_regex=False),                                            # no regex at all
    lambda j: j.update(pre_tokenizer={"type": "Sequence", "pretokenizers": [                         # StarCoder
        {"type": "Digits", "individual_digits": True}, j["pre_tokenizer"]]}),
    lambda j: j.update(pre_tokenizer={"type": "Sequence", "pretokenizers": [j["pre_tokenizer"], j["pre_tokenizer"]]}),
    lambda j: j.update(normalizer={"type": "NFC"}),
    lambda j: j["added_tokens"].append(dict(j["added_tokens"][0], id=9999, content="<|x|>", normalized=False)),   # mixed normalized
    lambda j: j["added_tokens"][0].update(rstrip=True),
])
def test_unsupported_gpt2_style_configurations_are_refused(tmp_path, mutate):
    j = json.load(open(GPT2))
    mutate(j)
    with pytest.raises(ValueError):
        HuggingFaceTokenizer(_host(), "unknown", _write(tmp_path, j))


def test_ex_loaders_refuse_an_unknown_pretokenizer():
    h = _host()
    L = _lib.load()
    toks = [bytes([b]) for b in range(256)]
    blob = np.frombuffer(b"".join(toks), np.uint8).copy()
    offs = np.arange(257, dtype=np.uint32)
    ids = np.arange(256, dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    calls = [
        lambda pt, err: L.smgx_tokenizer_load_tiktoken_file_ex(h.p, b"m", VOCAB.encode(), None, None, 0, pt, C.byref(err)),
        lambda pt, err: L.smgx_tokenizer_load_tiktoken_ex(h.p, b"m", p(blob), p(offs), p(ids), 256, None, None, 0, pt, C.byref(err)),
        lambda pt, err: L.smgx_tokenizer_load_bpe_merges_ex(h.p, b"m", p(blob), p(offs), p(ids), 256, None, 0, 0, None, None, 0, pt, C.byref(err)),
    ]
    for call in calls:
        err = C.c_char_p()
        assert call(7, err) == _lib.INVALID_ARGUMENT and b"pretokenizer" in err.value
        L.smgx_free_string(C.cast(err, C.c_void_p))
        for pt in (_lib.PRETOK_CL100K, _lib.PRETOK_R50K):
            err = C.c_char_p()
            assert call(pt, err) == _lib.SUCCESS, err.value
