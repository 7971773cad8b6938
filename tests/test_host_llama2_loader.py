"""CPU only: loading SentencePiece-style tokenizer.json files (Llama 2, Mistral, TinyLlama) on a host-mirror policy (device_id = -1): the
legacy Prepend + Replace shape and the Metaspace variants, read as the live `tokenizers` crate reads them; the shapes that stay refused;
and the argument checks of smgx_tokenizer_load_bpe_metaspace.  Encoding needs the GPU (tests/test_gpu_tokenizer_llama2.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from smg_b200 import SmgxError, _lib
from smg_b200.policy import CacheAwareConfig, HuggingFaceTokenizer, _Handle, _hf_sentencepiece

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIXTURE = os.path.join(GOLD, "hf_llama2_style_tokenizer.json")
SCHEMES = {"never": _lib.PREPEND_NEVER, "first": _lib.PREPEND_FIRST, "always": _lib.PREPEND_ALWAYS}


def _fixture(**top):
    j = json.load(open(FIXTURE))
    j.update(top)
    return j


def _metaspace(**keys):
    return _fixture(normalizer=None, pre_tokenizer={"type": "Metaspace", "replacement": "▁", **keys})


def _load(tmp_path, j):
    (tmp_path / "t.json").write_text(json.dumps(j))
    return HuggingFaceTokenizer(_Handle(CacheAwareConfig(eviction_interval_secs=0), -1), "unknown", str(tmp_path / "t.json"))


ACCEPTED = [
    {}, {"prepend_scheme": "first", "split": False}, {"prepend_scheme": "always", "split": False}, {"prepend_scheme": "first", "split": True},
    {"prepend_scheme": "never", "split": False}, {"prepend_scheme": "never", "split": True}, {"prepend_scheme": "always"},
    {"add_prefix_space": True}, {"add_prefix_space": True, "split": False}, {"add_prefix_space": True, "prepend_scheme": "first"},
    {"add_prefix_space": False, "prepend_scheme": "never"}, {"str_rep": "▁", "add_prefix_space": True, "split": False},
]


def test_legacy_shape_loads_and_encode_fails_loudly_without_device(tmp_path):
    tok = _load(tmp_path, _fixture())
    assert tok.growth == 2
    assert _hf_sentencepiece(_fixture()) == (_lib.SP_LEGACY, _lib.PREPEND_ALWAYS, 0)
    with pytest.raises(SmgxError):
        tok.encode("héllo wörld")


@pytest.mark.parametrize("keys", ACCEPTED)
def test_metaspace_variants_load_as_tokenizers_reads_them(tmp_path, keys):
    """Each key set is deserialized by the installed `tokenizers`; its canonical form (prepend_scheme, split) is what the loader hands
    to the ABI."""
    tk = pytest.importorskip("tokenizers")
    j = _metaspace(**keys)
    canon = json.loads(tk.Tokenizer.from_str(json.dumps(j)).to_str())["pre_tokenizer"]
    assert _hf_sentencepiece(j) == (_lib.SP_METASPACE, SCHEMES[canon["prepend_scheme"]], int(canon["split"]))
    tok = _load(tmp_path, j)
    assert tok.growth == 2
    with pytest.raises(SmgxError):
        tok.encode("héllo wörld")


def test_add_prefix_space_false_needs_prepend_scheme_never(tmp_path):
    """`tokenizers` refuses add_prefix_space = false unless prepend_scheme is "never"; so does the loader."""
    tk = pytest.importorskip("tokenizers")
    for keys in ({"add_prefix_space": False}, {"add_prefix_space": False, "prepend_scheme": "always"}):
        with pytest.raises(Exception):
            tk.Tokenizer.from_str(json.dumps(_metaspace(**keys)))
        with pytest.raises(ValueError):
            _load(tmp_path, _metaspace(**keys))


def _drop_vocab(tok):
    def f(j):
        del j["model"]["vocab"][tok]
        j["model"]["merges"] = [m for m in j["model"]["merges"] if tok not in m and "".join(m) != tok]
    return f


def _bad_merge(j):
    v = j["model"]["vocab"]
    for t in ("x", "▁x", "x▁x"):
        v.setdefault(t, len(v))
    j["model"]["merges"].append(["x", "▁x"])


def _set(path, value):
    def f(j):
        d = j
        for k in path[:-1]:
            d = d[k]
        d[path[-1]] = value
    return f


REFUSED = {
    "missing <0x41>": _drop_vocab("<0x41>"),
    "missing ▁": _drop_vocab("▁"),
    "ignore_merges": _set(["model", "ignore_merges"], True),
    "dropout": _set(["model", "dropout"], 0.1),
    "byte_fallback false": _set(["model", "byte_fallback"], False),
    "continuing_subword_prefix": _set(["model", "continuing_subword_prefix"], "##"),
    "end_of_word_suffix": _set(["model", "end_of_word_suffix"], "</w>"),
    "Prepend alone": _set(["normalizer"], {"type": "Prepend", "prepend": "▁"}),
    "Replace alone": _set(["normalizer"], {"type": "Replace", "pattern": {"String": " "}, "content": "▁"}),
    "Replace of a tab": _set(["normalizer", "normalizers", 1, "pattern"], {"String": "\t"}),
    "Replace by regex": _set(["normalizer", "normalizers", 1, "pattern"], {"Regex": " "}),
    "Prepend of another string": _set(["normalizer", "normalizers", 0, "prepend"], "_"),
    "legacy with a pre_tokenizer": _set(["pre_tokenizer"], {"type": "Metaspace", "replacement": "▁"}),
    "normalized specials with the legacy normalizer": lambda j: [a.update(normalized=True) for a in j["added_tokens"]],
    "lstrip": lambda j: j["added_tokens"][3].update(lstrip=True),
    "mixed normalized": lambda j: j["added_tokens"][0].update(normalized=True),
    "not BPE": _set(["model", "type"], "Unigram"),
}
REFUSED_METASPACE = {
    "replacement _": {"replacement": "_"},
    "unknown prepend_scheme": {"prepend_scheme": "sometimes"},
    "split as a string": {"split": "false"},
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_unsupported_files_are_refused(tmp_path, name):
    j = _fixture()
    REFUSED[name](j)
    with pytest.raises(ValueError):
        _load(tmp_path, j)


@pytest.mark.parametrize("name", sorted(REFUSED_METASPACE))
def test_unsupported_metaspace_keys_are_refused(tmp_path, name):
    with pytest.raises(ValueError):
        _load(tmp_path, _metaspace(**REFUSED_METASPACE[name]))
    with pytest.raises(ValueError):   # a Metaspace pre_tokenizer together with a normalizer
        _load(tmp_path, _fixture(pre_tokenizer={"type": "Metaspace", "replacement": "▁", "prepend_scheme": "first", "split": False}))


def test_merge_that_straddles_a_cut_is_refused_by_name(tmp_path):
    """("x", "▁x") would join a piece ending in x to the next one starting with ▁: no cut at ▁ is exact then.  With split = true the cut
    before every ▁ is the semantics, and the same vocabulary loads."""
    j = _fixture()
    _bad_merge(j)
    with pytest.raises(ValueError, match='"x", "▁x"'):
        _load(tmp_path, j)
    j = _metaspace(prepend_scheme="first", split=False)
    _bad_merge(j)
    with pytest.raises(ValueError, match='"x", "▁x"'):
        _load(tmp_path, j)
    j = _metaspace(prepend_scheme="first", split=True)
    _bad_merge(j)
    assert _load(tmp_path, j).growth == 2


def test_abi_checks_pointers_and_modes():
    h, L = _Handle(CacheAwareConfig(eviction_interval_secs=0), -1), _lib.load()
    j = _fixture()
    vocab = j["model"]["vocab"]
    toks = [s.encode() for s in vocab]
    blob = np.frombuffer(b"".join(toks), dtype=np.uint8).copy()
    offs = np.zeros(len(toks) + 1, np.uint32)
    np.cumsum([len(t) for t in toks], out=offs[1:])
    ids = np.asarray(list(vocab.values()), np.uint32)
    mg = np.asarray([vocab[t] for m in j["model"]["merges"] for t in m], np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731

    def load(blob_p=p(blob), offs_p=p(offs), ids_p=p(ids), mg_p=p(mg), shape=_lib.SP_LEGACY, scheme=_lib.PREPEND_ALWAYS, split=0):
        err = C.c_char_p()
        st = L.smgx_tokenizer_load_bpe_metaspace(h.p, b"m", blob_p, offs_p, ids_p, len(toks), mg_p, len(mg) // 2, None, None, 0,
                                                 shape, scheme, split, C.byref(err))
        msg = err.value
        if msg is not None:
            L.smgx_free_string(C.cast(err, C.c_void_p))
        return st, msg
    assert load() == (_lib.SUCCESS, None)
    for scheme in SCHEMES.values():
        for split in (0, 1):
            assert load(shape=_lib.SP_METASPACE, scheme=scheme, split=split) == (_lib.SUCCESS, None)
    for kw, word in (({"blob_p": None}, b"null"), ({"offs_p": None}, b"null"), ({"ids_p": None}, b"null"), ({"mg_p": None}, b"null"),
                     ({"shape": 2}, b"shape"), ({"shape": -1}, b"shape"), ({"shape": 1, "scheme": 3}, b"prepend_scheme"),
                     ({"shape": 1, "scheme": -1}, b"prepend_scheme"), ({"shape": 1, "split": 2}, b"split"),
                     ({"scheme": _lib.PREPEND_FIRST}, b"legacy"), ({"split": 1}, b"legacy")):
        st, msg = load(**kw)
        assert st == _lib.INVALID_ARGUMENT and msg and word in msg, (kw, msg)
    assert L.smgx_tokenizer_load_bpe_metaspace(None, b"m", p(blob), p(offs), p(ids), len(toks), p(mg), len(mg) // 2, None, None, 0, 0, 2, 0,
                                               None) == _lib.INVALID_ARGUMENT
