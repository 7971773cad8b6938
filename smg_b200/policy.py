"""Host-side mirror of the reference's plugin surface for the cache-aware path, over the smgx C ABI.

Names, argument meaning and error behaviour follow the reference so the parity tests read like its own tests:
  * CacheAwareConfig / SelectWorkerInfo / LoadBalancingPolicy   model_gateway/src/policies/mod.rs:43-175
  * CacheAwarePolicy                                            model_gateway/src/policies/cache_aware.rs
  * PolicyFactory                                               model_gateway/src/policies/factory.rs:17-93
  * PositionalIndexer                                           crates/kv_index/src/event_tree.rs:257-760
  * KvEventMonitor (get_indexer / block_size / set_block_size)  model_gateway/src/worker/kv_event_monitor.rs
  * the Worker scalars the path reads                           model_gateway/src/worker/worker.rs:109-230
Every decision comes out of the CUDA kernels; this file only marshals arrays.
"""
import ctypes as C
from dataclasses import dataclass
from typing import List, Mapping, Optional, Sequence

import numpy as np

from . import _lib

UNKNOWN_MODEL_ID = "unknown"


def normalize_model_key(model_id: str) -> str:  # policies/mod.rs:151-157
    return model_id if model_id else UNKNOWN_MODEL_ID


@dataclass
class CacheAwareConfig:  # policies/mod.rs:94-117
    cache_threshold: float = 0.5
    balance_abs_threshold: int = 32
    balance_rel_threshold: float = 1.1
    eviction_interval_secs: int = 30
    max_tree_size: int = 10000
    block_size: int = 16


@dataclass
class SelectWorkerInfo:  # policies/mod.rs:161-175 (headers are read by consistent_hashing only; hash_ring by prefix_hash and consistent_hashing)
    request_text: Optional[str] = None
    tokens: Optional[Sequence[int]] = None
    hash_ring: Optional["HashRing"] = None
    headers: Optional[Mapping] = None   # header name (any case) → value (str or bytes, or a list whose first item HeaderMap::get returns)


class BasicWorker:
    """The scalars CacheAwarePolicy reads through `trait Worker` (worker/worker.rs:114,151-153,187,208,217)."""

    def __init__(self, url: str, model_id: str = ""):
        self._url, self._model_id = url, model_id
        self._load, self._healthy, self._circuit_ok, self._processed = 0, True, True, 0

    def url(self): return self._url
    def model_id(self): return self._model_id
    def load(self): return self._load
    def is_healthy(self): return self._healthy
    def circuit_breaker_can_execute(self): return self._circuit_ok
    def increment_processed(self): self._processed = getattr(self, "_processed", 0) + 1
    def processed(self): return getattr(self, "_processed", 0)
    def processed(self): return self._processed
    def increment_load(self): self._load += 1
    def decrement_load(self): self._load = max(0, self._load - 1)
    def set_load(self, v): self._load = int(v)
    def set_healthy(self, ok: bool): self._healthy = bool(ok)      # set_status(Ready) ⇔ True; any other status ⇔ False
    def set_circuit_ok(self, ok: bool): self._circuit_ok = bool(ok)


def _u32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint32))


def _u64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint64))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and a.size else None


class _Handle:
    """Owns one smgx_policy*."""

    def __init__(self, cfg: CacheAwareConfig, device_id: int, max_batch: int = 0, max_tokens_per_request: int = 0, tree_batch_mode: int = 0):
        self.L = _lib.load()
        c = _lib.Config()
        self.L.smgx_default_config(C.byref(c))
        c.cache_threshold, c.balance_abs_threshold = cfg.cache_threshold, cfg.balance_abs_threshold
        c.balance_rel_threshold, c.eviction_interval_secs = cfg.balance_rel_threshold, cfg.eviction_interval_secs
        c.max_tree_size, c.block_size = cfg.max_tree_size, cfg.block_size
        c.device_id, c.max_batch, c.max_tokens_per_request = device_id, max_batch, max_tokens_per_request
        c.tree_batch_mode = tree_batch_mode
        err = _lib.new_err()
        self.p = self.L.smgx_policy_create(C.byref(c), C.byref(err))
        if not self.p:
            _lib.check(_lib.UNKNOWN_ERROR if not err.value else _lib.DEVICE_ERROR, err)
        self.device_id = device_id

    def close(self):
        if getattr(self, "p", None):
            self.L.smgx_policy_free(self.p)
            self.p = None

    def __del__(self):
        self.close()

    def call(self, fn, *args):
        err = _lib.new_err()
        code = getattr(self.L, fn)(self.p, *args, C.byref(err))
        _lib.check(code, err)


class ApplyError(Exception):  # kv_index::ApplyError (event_tree.rs:88-106)
    pass


class PositionalIndexer:
    """kv_index::PositionalIndexer bound to (policy handle, model).  Blocks are (seq_hash, content_hash) pairs =
    StoredBlock (event_tree.rs:81-86); the caller-owned WorkerBlockMap lives inside the library per worker id."""

    def __init__(self, handle: _Handle, model: str, jump_size: int = 32):
        if jump_size <= 0:
            raise ValueError("jump_size must be greater than 0")  # event_tree.rs:280
        self.h, self.model = handle, model.encode()
        self.h.call("smgx_indexer_create", self.model, jump_size)

    @classmethod
    def standalone(cls, jump_size: int = 32, device_id: int = 0):
        """An indexer with a private policy handle (the reference constructs PositionalIndexer::new(jump) directly)."""
        if jump_size <= 0:
            raise ValueError("jump_size must be greater than 0")
        return cls(_Handle(CacheAwareConfig(eviction_interval_secs=0), device_id), UNKNOWN_MODEL_ID, jump_size)

    def intern_worker(self, url: str) -> int:
        out = C.c_uint32()
        self.h.call("smgx_indexer_intern_worker", self.model, url.encode(), C.byref(out))
        return out.value

    def worker_id(self, url: str) -> Optional[int]:
        out = C.c_int64()
        self.h.call("smgx_indexer_worker_id", self.model, url.encode(), C.byref(out))
        return None if out.value < 0 else out.value

    def apply_stored(self, worker_id: int, blocks, parent: Optional[int] = None):
        seq, con = _u64([b[0] for b in blocks]), _u64([b[1] for b in blocks])
        par = C.c_uint64(parent) if parent is not None else None
        try:
            self.h.call("smgx_indexer_apply_stored", self.model, worker_id, _p(seq), _p(con), len(blocks),
                        C.cast(C.byref(par), C.c_void_p) if par is not None else None)
        except _lib.SmgxError as e:
            if e.code == _lib.WORKER_NOT_TRACKED:
                raise ApplyError("WorkerNotTracked: " + e.msg)
            if e.code == _lib.PARENT_BLOCK_NOT_FOUND:
                raise ApplyError("ParentBlockNotFound: " + e.msg)
            raise

    def apply_stored_tokens(self, worker_id: int, seq_hashes, token_ids, block_size: int, parent: Optional[int] = None):
        seq, tok = _u64(seq_hashes), _u32(token_ids)
        par = C.c_uint64(parent) if parent is not None else None
        try:
            self.h.call("smgx_indexer_apply_stored_tokens", self.model, worker_id, _p(seq), _p(tok), block_size, seq.size,
                        C.cast(C.byref(par), C.c_void_p) if par is not None else None)
        except _lib.SmgxError as e:
            if e.code == _lib.WORKER_NOT_TRACKED:
                raise ApplyError("WorkerNotTracked: " + e.msg)
            if e.code == _lib.PARENT_BLOCK_NOT_FOUND:
                raise ApplyError("ParentBlockNotFound: " + e.msg)
            raise

    def apply_removed(self, worker_id: int, seq_hashes):
        s = _u64(seq_hashes)
        self.h.call("smgx_indexer_apply_removed", self.model, worker_id, _p(s), s.size)

    def apply_cleared(self, worker_id: int):
        self.h.call("smgx_indexer_apply_cleared", self.model, worker_id)

    def remove_worker(self, worker_id: int):
        self.h.call("smgx_indexer_remove_worker", self.model, worker_id)

    def current_size(self) -> int:
        out = C.c_uint64()
        self.h.call("smgx_indexer_current_size", self.model, C.byref(out))
        return out.value

    def entry_count(self) -> int:
        out = C.c_uint64()
        self.h.call("smgx_indexer_entry_count", self.model, C.byref(out))
        return out.value

    def find_matches(self, content_hashes, early_exit: bool = False):
        """→ (scores, tree_sizes) dicts keyed by worker id, like OverlapScores (event_tree.rs:112-118).  GPU kernel."""
        hs = _u64(content_hashes)
        cap = 2048
        sc, ts, nw = np.zeros(cap, np.uint32), np.zeros(cap, np.uint64), C.c_uint32()
        self.h.call("smgx_indexer_find_matches", self.model, _p(hs), hs.size, 1 if early_exit else 0, _p(sc), _p(ts), cap, C.byref(nw))
        ids = [i for i in range(nw.value) if sc[i] > 0]
        return {i: int(sc[i]) for i in ids}, {i: int(ts[i]) for i in ids}


class KvEventMonitor:
    """The slice of worker::KvEventMonitor the policy reads: per-model indexers and learned block sizes."""

    def __init__(self, policy: "CacheAwarePolicy", default_block_size: Optional[int] = None):
        self.policy, self.default_block_size, self.indexers = policy, default_block_size, {}
        self._learned = {}

    def create_indexer(self, model: str, jump_size: int = 64) -> PositionalIndexer:  # DEFAULT_JUMP_SIZE kv_event_monitor.rs:31
        ix = PositionalIndexer(self.policy._h, model, jump_size)
        self.indexers[model] = ix
        return ix

    def get_indexer(self, model: str) -> Optional[PositionalIndexer]:
        return self.indexers.get(model)

    def set_block_size(self, model: str, block_size: int):
        self.policy._h.call("smgx_indexer_set_block_size", model.encode(), block_size)

    def apply_events(self, model: str, worker_id: int, events):
        """One KvEventBatch of a worker's stream (kv_event_monitor.rs:513-517, apply_event :525-597) through smgx_kv_events_apply.
        `events`: dicts shaped like the proto — {"stored": {"blocks": [{"block_hash", "token_ids", "block_size"}...],
        "parent_block_hash": int | None}}, {"removed": {"block_hashes": [...]}} or {"cleared": {}}.  The first stored block with
        block_size > 0 teaches the model's block size once (learn_block_size :270-296).  Returns the number of fresh-chain fallbacks."""
        evs, hashes, toks, offs = [], [], [], [0]
        for ev in events:
            if "stored" in ev:
                st = ev["stored"]
                blocks = st.get("blocks", [])
                if blocks and not self._learned.get(model) and blocks[0].get("block_size", 0) > 0:
                    self.set_block_size(model, int(blocks[0]["block_size"]))
                    self._learned[model] = True
                parent = st.get("parent_block_hash")
                evs.append((0, len(hashes), len(blocks), 0 if parent is None else int(parent), 0 if parent is None else 1))
                for b in blocks:
                    hashes.append(int(b["block_hash"]))
                    toks.extend(int(t) for t in b.get("token_ids", []))
                    offs.append(len(toks))
            elif "removed" in ev:
                hs = [int(h) for h in ev["removed"].get("block_hashes", [])]
                evs.append((1, len(hashes), len(hs), 0, 0))
                for h in hs:
                    hashes.append(h)
                    offs.append(len(toks))
            elif "cleared" in ev:
                evs.append((2, 0, 0, 0, 0))
        arr = (_lib.KvEvent * max(len(evs), 1))()
        for i, (k, fb, nb, par, hp) in enumerate(evs):
            arr[i].kind, arr[i].worker_id, arr[i].first_block, arr[i].n_blocks = k, worker_id, fb, nb
            arr[i].parent_block_hash, arr[i].has_parent = par, hp
        h64 = np.ascontiguousarray(np.asarray([x if x < 2**63 else x - 2**64 for x in hashes] or [0], dtype=np.int64))
        t32, o32 = _u32(toks), _u32(offs)
        fallbacks = C.c_uint32()
        self.policy._h.call("smgx_kv_events_apply", model.encode(), C.cast(arr, C.c_void_p), len(evs), _p(h64), _p(o32), _p(t32) if t32.size else None,
                            len(hashes), C.byref(fallbacks))
        return fallbacks.value


class TokenMatchResult:  # kv_index::PrefixMatchResult (token_tree.rs:137-144)
    def __init__(self, tenant, matched, inp):
        self.tenant, self.matched_token_count, self.input_token_count = tenant, matched, inp


LRU, LFU, FIFO, MRU, FILO, PRIORITY = range(6)   # kv_index::EvictionPolicy (token_tree.rs:60-75)


class TokenTree:
    """kv_index::TokenTree bound to (policy handle, model): mutations on the host-authoritative tree inside the library,
    match_prefix_with_counts on the GPU mirror."""

    def __init__(self, handle: _Handle, model: str = UNKNOWN_MODEL_ID, policy: int = LRU):
        self.h, self.model = handle, model.encode()
        self.h.call("smgx_tree_create", self.model, policy)

    @classmethod
    def standalone(cls, policy: int = LRU, device_id: int = 0):
        return cls(_Handle(CacheAwareConfig(eviction_interval_secs=0), device_id), UNKNOWN_MODEL_ID, policy)

    def insert_tokens(self, tokens, tenant: str):
        t = _u32(tokens)
        self.h.call("smgx_tree_insert_tokens", self.model, _p(t), t.size, tenant.encode())

    def match_prefix_with_counts(self, tokens) -> TokenMatchResult:
        t = _u32(tokens)
        m, n = C.c_uint32(), C.c_uint32()
        buf = C.create_string_buffer(1024)
        self.h.call("smgx_tree_match_tokens", self.model, _p(t), t.size, C.byref(m), C.byref(n), C.cast(buf, C.c_void_p), 1024)
        return TokenMatchResult(buf.value.decode(), m.value, n.value)

    def evict_tenant(self, tenant: str, max_tokens: int):
        self.h.call("smgx_tree_evict_tenant", self.model, tenant.encode(), max_tokens)

    def evict_tenant_by_size(self, max_size: int):
        self.h.call("smgx_evict_cache", max_size)

    def tenant_token_size(self, tenant: str) -> int:
        out = C.c_uint64()
        self.h.call("smgx_tree_tenant_size", self.model, tenant.encode(), C.byref(out))
        return out.value

    def clear(self):
        self.h.call("smgx_tree_clear", self.model)

    def entries(self):
        out = C.c_void_p()
        self.h.call("smgx_tree_entries", self.model, C.byref(out))
        text = C.cast(out, C.c_char_p).value.decode()
        self.h.L.smgx_free_string(out)
        res = []
        for line in text.split("\n"):
            if not line:
                continue
            toks, tens = line.split("|")
            res.append(([int(x) for x in toks.split(",")] if toks else [],
                        [(kv.rsplit("=", 1)[0], int(kv.rsplit("=", 1)[1])) for kv in tens.split(";") if kv]))
        return res


class StringMatchResult:  # kv_index::PrefixMatchResult of the string tree (string_tree.rs:47-54)
    def __init__(self, tenant, matched, inp):
        self.tenant, self.matched_char_count, self.input_char_count = tenant, matched, inp


class Tree:
    """kv_index::Tree (char-level string tree, HTTP text routing) bound to (policy handle, model): mutations on the
    host-authoritative tree inside the library, match_prefix_with_counts on the GPU mirror."""

    def __init__(self, handle: _Handle, model: str = UNKNOWN_MODEL_ID):
        self.h, self.model = handle, model.encode()

    @classmethod
    def standalone(cls, device_id: int = 0):
        return cls(_Handle(CacheAwareConfig(eviction_interval_secs=0), device_id), UNKNOWN_MODEL_ID)

    @staticmethod
    def _b(text: str):
        b = text.encode("utf-8")
        return (np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, np.uint8)), len(b)

    def insert_text(self, text: str, tenant: str):
        a, n = self._b(text)
        self.h.call("smgx_stree_insert_text", self.model, _p(a), n, tenant.encode())

    def match_prefix_with_counts(self, text: str) -> StringMatchResult:
        a, n = self._b(text)
        m, k = C.c_uint32(), C.c_uint32()
        buf = C.create_string_buffer(1024)
        self.h.call("smgx_stree_match", self.model, _p(a), n, C.byref(m), C.byref(k), C.cast(buf, C.c_void_p), 1024)
        return StringMatchResult(buf.value.decode(), m.value, k.value)

    def prefix_match_tenant(self, text: str, tenant: str) -> str:
        a, n = self._b(text)
        out = C.c_uint32()
        self.h.call("smgx_stree_prefix_match_tenant", self.model, _p(a), n, tenant.encode(), C.byref(out))
        return text.encode("utf-8")[: out.value].decode("utf-8")

    def evict_tenant_by_size(self, max_size: int):
        self.h.call("smgx_evict_cache", max_size)

    def _sizes(self, maintained: int):
        out = C.c_void_p()
        self.h.call("smgx_stree_sizes", self.model, maintained, C.byref(out))
        text = C.cast(out, C.c_char_p).value.decode()
        self.h.L.smgx_free_string(out)
        res = {}
        for line in text.split("\n"):
            if line:
                k, v = line.rsplit("=", 1)
                res[k] = int(v)
        return res

    def get_used_size_per_tenant(self):
        return self._sizes(0)

    def get_tenant_char_count(self):
        return self._sizes(1)

    def node_count(self) -> int:
        out = C.c_uint64()
        self.h.call("smgx_stree_node_count", self.model, C.byref(out))
        return out.value

    def clear(self):
        self.h.call("smgx_stree_clear", self.model)

    # -- mesh wire format: kv_index::snapshot::TreeSnapshot, bincode (snapshot.rs; string_tree.rs:1052-1578) --
    def snapshot_bytes(self) -> bytes:  # Tree::snapshot().to_bytes()
        out, ln = C.c_void_p(), C.c_uint64()
        self.h.call("smgx_stree_snapshot", self.model, C.byref(out), C.byref(ln))
        raw = C.string_at(out, ln.value)
        self.h.L.smgx_free_string(out)
        return raw

    @classmethod
    def from_snapshot_bytes(cls, data: bytes, device_id: int = 0):  # TreeSnapshot::from_bytes + Tree::from_snapshot (:1228)
        t = cls.standalone(device_id)
        t.h.call("smgx_stree_load_snapshot", t.model, data, len(data))
        return t

    def merge_snapshot_bytes(self, data: bytes):  # Tree::merge_snapshot (:1318)
        self.h.call("smgx_stree_merge_snapshot", self.model, data, len(data))

    def entries(self):
        out, ln = C.c_void_p(), C.c_uint64()
        self.h.call("smgx_stree_entries", self.model, C.byref(out), C.byref(ln))
        raw = C.string_at(out, ln.value).decode("utf-8")
        self.h.L.smgx_free_string(out)
        res = []
        for rec in raw.split("\x1e"):
            if not rec:
                continue
            path, tens = rec.split("\x1f")
            res.append((path, [(kv.rsplit("=", 1)[0], int(kv.rsplit("=", 1)[1])) for kv in tens.split(";") if kv]))
        return res


# The reference's TiktokenModel set (tiktoken.rs:136-184) → the pre-tokenizer regex of the encoding.  r50k_base, p50k_base and
# p50k_edit all split text with tiktoken's GPT-2 pattern; they differ only in vocabulary and specials, which the caller supplies.
TIKTOKEN_ENCODINGS = {"cl100k_base": _lib.PRETOK_CL100K, "r50k_base": _lib.PRETOK_R50K, "p50k_base": _lib.PRETOK_R50K, "p50k_edit": _lib.PRETOK_R50K}


class TiktokenTokenizer:
    """tokenizer::TiktokenTokenizer (crates/tokenizer/src/tiktoken.rs:132) on the GPU, bound to (policy handle, model).
    encode() keeps the reference's behaviour of always recognising special-token strings (tiktoken.rs:444-462).
    `encoding` names the tiktoken encoding whose pre-tokenizer regex is used (TIKTOKEN_ENCODINGS)."""

    def __init__(self, handle: _Handle, model: str, path: str, special_tokens=None, encoding: str = "cl100k_base"):
        if encoding not in TIKTOKEN_ENCODINGS:
            raise ValueError(f"unknown tiktoken encoding {encoding!r}; supported: {', '.join(TIKTOKEN_ENCODINGS)}")
        self.h, self.model = handle, model.encode()
        self.growth = 1   # most tokens per byte of text: smgx_tokenize_batch's cap_tokens rule
        sp = list((special_tokens or {}).items())
        strs = (C.c_char_p * max(len(sp), 1))(*[k.encode() for k, _ in sp]) if sp else None
        ids = _u32([v for _, v in sp])
        self.h.call("smgx_tokenizer_load_tiktoken_file_ex", self.model, path.encode(), strs, _p(ids), len(sp), TIKTOKEN_ENCODINGS[encoding])

    @staticmethod
    def _ragged(texts):
        blobs = [t.encode("utf-8") for t in texts]
        offsets = np.zeros(len(blobs) + 1, dtype=np.uint32)
        np.cumsum([len(b) for b in blobs], out=offsets[1:])
        data = np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8).copy()
        return data, offsets

    def encode_batch(self, texts, add_special_tokens: bool = False):
        data, offsets = self._ragged(texts)
        n = len(texts)
        cap = self.growth * int(offsets[-1]) + 1
        out, toff = np.zeros(cap, np.uint32), np.zeros(n + 1, np.uint32)
        self.h.call("smgx_tokenize_batch", self.model, _p(data), _p(offsets), n, _p(out), _p(toff), cap)
        return [out[toff[i]:toff[i + 1]].tolist() for i in range(n)]

    def encode(self, text: str, add_special_tokens: bool = False):
        return self.encode_batch([text])[0]


LLAMA3_SPLIT_PATTERN = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+")
# Qwen2 / Qwen2.5 / Qwen3 / QwQ: the Llama-3 pattern with \p{N} in place of \p{N}{1,3} (every digit is a piece of its own)
QWEN2_SPLIT_PATTERN = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+")
_SPLIT_PATTERNS = {LLAMA3_SPLIT_PATTERN: _lib.PRETOK_CL100K, QWEN2_SPLIT_PATTERN: _lib.PRETOK_QWEN2}
# DeepSeek V2 / V2.5 / Coder-V2 / V3 / V3.1 / R1: three Isolated Splits chained — digit triples, kana/CJK runs (U+4E00-U+9FA5,
# U+3040-U+30FF), then words with punctuation — as the JSON strings of their tokenizer.json decode (the CR and LF are literal characters).
DEEPSEEK_SPLIT_PATTERNS = (
    "\\p{N}{1,3}",
    "[一-龥぀-ゟ゠-ヿ]+",
    "[!\"#$%&'()*+,\\-./:;<=>?@\\[\\\\\\]^_`{|}~][A-Za-z]+|[^\r\n\\p{L}\\p{P}\\p{S}]?[\\p{L}\\p{M}]+| ?[\\p{P}\\p{S}]+[\r\n]*|\\s*[\r\n]+|"
    "\\s+(?!\\S)|\\s+")


def _byte_level_decoder():
    """Inverse of the GPT-2 bytes_to_unicode table used by `tokenizers`' ByteLevel pre-tokenizer (pre_tokenizers/byte_level.rs)."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("\xa1"), ord("\xac") + 1)) + list(range(ord("\xae"), ord("\xff") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return {chr(c): b for b, c in zip(bs, cs)}


def _hf_pretokenizer(pre):
    """tokenizer.json `pre_tokenizer` → smgx_pretokenizer, or ValueError for a shape the GPU path does not implement.  Three shapes:
    Split(Llama-3 / cl100k regex or Qwen2 regex, Isolated) + ByteLevel(use_regex=False), and GPT-2's ByteLevel(use_regex=True,
    add_prefix_space=False) alone or as a one-element Sequence (its built-in regex is tiktoken's r50k pattern)."""
    steps = pre.get("pretokenizers", [pre]) if pre.get("type") == "Sequence" else [pre]
    kinds = [s.get("type") for s in steps]
    if kinds == ["ByteLevel"]:
        bl = steps[0]
        if bl.get("use_regex", True) is True and bl.get("add_prefix_space") is False:   # use_regex defaults to true in the crate
            return _lib.PRETOK_R50K
        raise ValueError("tokenizer.json: a lone ByteLevel pre_tokenizer must have use_regex=True and add_prefix_space=False")
    split = [s for s in steps if s.get("type") == "Split"]
    bl = [s for s in steps if s.get("type") == "ByteLevel"]
    if kinds != ["Split", "ByteLevel"] or split[0].get("pattern", {}).get("Regex") not in _SPLIT_PATTERNS or \
            str(split[0].get("behavior")).lower() != "isolated" or split[0].get("invert") or bl[0].get("use_regex") or bl[0].get("add_prefix_space"):
        raise ValueError("tokenizer.json: pre_tokenizer must be Split(Llama-3 or Qwen2 regex, Isolated) + ByteLevel(use_regex=False), "
                         "or ByteLevel(use_regex=True, add_prefix_space=False) alone")
    return _SPLIT_PATTERNS[split[0]["pattern"]["Regex"]]


def _hf_deepseek_pretokenizer(pre):
    """True for DeepSeek's pre_tokenizer, Sequence[Split(DEEPSEEK_SPLIT_PATTERNS[0]), Split([1]), Split([2]), ByteLevel], every Split
    Isolated and not inverted, ByteLevel with use_regex = false and add_prefix_space = false (trim_offsets either way); False when the
    pre_tokenizer has fewer than two Splits; ValueError naming the difference for any other chain of Splits."""
    steps = pre.get("pretokenizers", []) if pre.get("type") == "Sequence" else [pre]
    kinds = [s.get("type") for s in steps]
    if kinds.count("Split") < 2:
        return False
    want = "Sequence[Split(\\p{N}{1,3}), Split(kana/CJK), Split(DeepSeek word regex), ByteLevel]"
    if kinds != ["Split", "Split", "Split", "ByteLevel"]:
        raise ValueError(f"tokenizer.json: a chain of Splits is supported only as DeepSeek's {want}, not {kinds}")
    for k, (s, pat) in enumerate(zip(steps, DEEPSEEK_SPLIT_PATTERNS)):
        if s.get("pattern") != {"Regex": pat}:
            raise ValueError(f"tokenizer.json: Split {k} of the chain has pattern {s.get('pattern')!r}; DeepSeek's {want} needs {pat!r}")
        if str(s.get("behavior")).lower() != "isolated" or s.get("invert"):
            raise ValueError(f"tokenizer.json: Split {k} of the chain must be Isolated with invert = false, not behavior "
                             f"{s.get('behavior')!r}, invert {s.get('invert')!r}")
    bl = steps[3]
    if bl.get("use_regex") is not False or bl.get("add_prefix_space") is not False:
        raise ValueError("tokenizer.json: the ByteLevel step of the DeepSeek chain must have use_regex = false and add_prefix_space = false")
    return True


def _overlapping_added_tokens(a, b):
    """A string of `a` and one of `b` that can overlap in a text (one inside the other, or a suffix of one that starts the other), or
    None.  `tokenizers` cuts added tokens marked normalized = false first and the others in what is left, so two such strings make the
    result depend on the marks even without a normalizer."""
    prefixes = lambda xs: {s[:k] for s in xs for k in range(1, len(s))}   # noqa: E731
    substrings = lambda xs: {s[i:k] for s in xs for i in range(len(s)) for k in range(i + 1, len(s) + 1)}   # noqa: E731
    for xs, ys in ((a, b), (b, a)):
        pre_ys, sub_ys = prefixes(ys), substrings(ys)
        for x in xs:
            if x in sub_ys:
                return x, next(y for y in ys if x in y)
            for k in range(1, len(x)):
                if x[k:] in pre_ys:
                    return x, next(y for y in ys if y.startswith(x[k:]))
    return None


def _hf_normalizer(norm):
    """tokenizer.json `normalizer` → smgx_normalizer: none, or NFC alone or as a one-element Sequence.  Every other normalizer is refused."""
    if norm is None:
        return _lib.NORMALIZER_NONE
    steps = norm.get("normalizers", []) if norm.get("type") == "Sequence" else [norm]
    if [s.get("type") for s in steps] == ["NFC"]:
        return _lib.NORMALIZER_NFC
    raise ValueError("tokenizer.json: the only normalizer supported on the GPU path is NFC (alone or as a one-element Sequence)")


METASPACE = "▁"   # ▁, SentencePiece's space
_PREPEND_SCHEMES = {"never": _lib.PREPEND_NEVER, "first": _lib.PREPEND_FIRST, "always": _lib.PREPEND_ALWAYS}


def _hf_sentencepiece(j):
    """The two SentencePiece-style tokenizer.json shapes → (smgx_sp_shape, smgx_prepend_scheme, split), or None when the file has neither
    the legacy normalizer nor a Metaspace pre_tokenizer.  A file that has one of them in any other form is refused with ValueError.
      legacy     normalizer Sequence[Prepend("▁"), Replace(String " " → "▁")], pre_tokenizer null (Llama 2, Mistral v0.1/v0.2, TinyLlama);
      metaspace  normalizer null, pre_tokenizer Metaspace(replacement "▁", prepend_scheme, split), read as the `tokenizers` crate reads it:
                 prepend_scheme defaults to "always", split to true, and add_prefix_space = false is only valid with prepend_scheme
                 "never" (which it then means)."""
    norm, pre = j.get("normalizer"), j.get("pre_tokenizer")
    steps = norm.get("normalizers", []) if norm and norm.get("type") == "Sequence" else [norm] if norm else []
    if any(s.get("type") in ("Prepend", "Replace") for s in steps):
        if [s.get("type") for s in steps] != ["Prepend", "Replace"]:
            return None   # e.g. Prepend alone: refused by _hf_normalizer
        p, r = steps
        if p.get("prepend") != METASPACE or r.get("pattern") != {"String": " "} or r.get("content") != METASPACE:
            raise ValueError("tokenizer.json: the SentencePiece-style normalizer must be Sequence[Prepend(\"▁\"), Replace(String \" \" → \"▁\")]")
        if pre is not None:
            raise ValueError("tokenizer.json: the Prepend + Replace normalizer is supported with pre_tokenizer null only")
        return _lib.SP_LEGACY, _lib.PREPEND_ALWAYS, 0
    if not pre or pre.get("type") != "Metaspace":
        return None
    if norm is not None:
        raise ValueError("tokenizer.json: a Metaspace pre_tokenizer is supported with normalizer null only")
    if pre.get("replacement") != METASPACE:
        raise ValueError("tokenizer.json: the Metaspace replacement must be \"▁\" (U+2581)")
    scheme = pre.get("prepend_scheme", "always")
    if scheme not in _PREPEND_SCHEMES:
        raise ValueError(f"tokenizer.json: unknown Metaspace prepend_scheme {scheme!r}")
    if pre.get("add_prefix_space") is False and scheme != "never":
        raise ValueError("tokenizer.json: Metaspace add_prefix_space = false does not match prepend_scheme " + repr(scheme))
    split = pre.get("split", True)
    if not isinstance(split, bool):
        raise ValueError("tokenizer.json: Metaspace split must be true or false")
    return _lib.SP_METASPACE, _PREPEND_SCHEMES[scheme], int(split)


class HuggingFaceTokenizer(TiktokenTokenizer):
    """tokenizer::HuggingFaceTokenizer (crates/tokenizer/src/huggingface.rs) for the BPE families the GPU path covers:
    - byte-level BPE: tokenizer.json with no normalizer or NFC, either Split(Llama-3 / cl100k or Qwen2 regex, Isolated) +
      ByteLevel(use_regex=False) or GPT-2's ByteLevel(use_regex=True, add_prefix_space=False) alone, model BPE without dropout / unk /
      byte_fallback;
    - DeepSeek V2 / V3 / R1 byte-level BPE: normalizer null or the identity Sequence[], pre_tokenizer the chain of three Splits
      (_hf_deepseek_pretokenizer) + ByteLevel(use_regex=False); added tokens may mix `normalized` marks when no two of them can overlap;
    - SentencePiece-style BPE (Llama 2, CodeLlama, Mistral, Mixtral, TinyLlama): the legacy normalizer Sequence[Prepend("▁"),
      Replace(" " → "▁")] without a pre_tokenizer, or Metaspace(replacement "▁") without a normalizer (_hf_sentencepiece); model BPE with
      byte_fallback = true, the 256 <0xXX> tokens and "▁" in the vocabulary, ignore_merges = false, no dropout / continuing_subword_prefix /
      end_of_word_suffix.  Vocabulary strings are raw UTF-8.  The load also refuses a vocabulary whose merges would not let the GPU cut a
      stretch into pieces at ▁ (smgx_tokenizer_load_bpe_metaspace); the message names the merge.
    Anything else is refused loudly with ValueError — there is no CPU tokenizer behind this."""

    def __init__(self, handle: _Handle, model: str, path: str):   # noqa: D401 — does not call the tiktoken loader
        import json
        self.h, self.model = handle, model.encode()
        j = json.load(open(path, encoding="utf-8"))
        mdl = j.get("model") or {}
        sp = _hf_sentencepiece(j)
        if sp is not None:
            self._load_sentencepiece(j, mdl, sp)
            return
        if mdl.get("type") != "BPE" or mdl.get("dropout") or mdl.get("unk_token") or mdl.get("byte_fallback") or \
                mdl.get("continuing_subword_prefix") or mdl.get("end_of_word_suffix"):
            raise ValueError("tokenizer.json: only plain byte-level BPE models are supported on the GPU path")
        deepseek = _hf_deepseek_pretokenizer(j.get("pre_tokenizer") or {})
        if deepseek:   # DeepSeek files carry the identity normalizer, an empty Sequence; it is accepted with this pre_tokenizer only
            if j.get("normalizer") not in (None, {"type": "Sequence", "normalizers": []}):
                raise ValueError("tokenizer.json: the DeepSeek pre_tokenizer is supported with normalizer null or an empty Sequence only")
            norm, pretok = _lib.NORMALIZER_NONE, _lib.PRETOK_DEEPSEEK
        else:
            norm = _hf_normalizer(j.get("normalizer"))
            pretok = _hf_pretokenizer(j.get("pre_tokenizer") or {})
        # NFC goes with the Qwen2 Split or GPT-2's ByteLevel; a Llama-3 Split with a normalizer stays refused, as before
        if norm != _lib.NORMALIZER_NONE and pretok == _lib.PRETOK_CL100K:
            raise ValueError("tokenizer.json: a normalizer is supported with the Qwen2 Split or GPT-2's ByteLevel pre_tokenizer, not the Llama-3 Split")
        dec = _byte_level_decoder()
        vocab = mdl["vocab"]
        toks = [bytes(dec[c] for c in s) for s in vocab]
        ids = _u32(list(vocab.values()))
        merges = []
        for mg in mdl.get("merges", []):
            a, b = mg.split(" ") if isinstance(mg, str) else mg
            merges += [vocab[a], vocab[b]]
        offs = np.zeros(len(toks) + 1, dtype=np.uint32)
        np.cumsum([len(t) for t in toks], out=offs[1:])
        blob = np.frombuffer(b"".join(toks), dtype=np.uint8).copy()
        strs, sp_ids, n_added = self._added_tokens(j, norm != _lib.NORMALIZER_NONE, mixed_ok=deepseek)
        self.growth = 3 if norm != _lib.NORMALIZER_NONE else 1   # NFC can grow text threefold
        mg = _u32(merges)
        self.h.call("smgx_tokenizer_load_bpe_merges_norm", self.model, _p(blob), _p(offs), _p(ids), len(toks), _p(mg), len(merges) // 2,
                    1 if mdl.get("ignore_merges") else 0, strs, _p(sp_ids), n_added, pretok, norm)

    @staticmethod
    def _added_tokens(j, normalizer: bool, mixed_ok: bool = False):
        """added_tokens → (C strings, ids, count) for the loaders, or ValueError for the kinds the GPU path does not implement.
        mixed_ok (DeepSeek's shape only): accept mixed `normalized` marks as long as no string of one mark can overlap one of the other."""
        added = [(a["content"], a["id"]) for a in j.get("added_tokens", [])]
        for a in j.get("added_tokens", []):
            if a.get("lstrip") or a.get("rstrip") or a.get("single_word"):
                raise ValueError("tokenizer.json: added tokens with lstrip / rstrip / single_word are not supported")
        # Without a normalizer, `tokenizers` extracts added tokens in one pass over the raw text whether they are marked normalized or
        # not, as long as all of them carry the same mark; a mix splits the text in two passes, which the GPU path does not implement.
        # The two passes give what one pass gives when no string of one mark overlaps a string of the other.
        marks = {bool(a.get("normalized", False)) for a in j.get("added_tokens", [])}
        if len(marks) > 1 and not mixed_ok:
            raise ValueError("tokenizer.json: added tokens with mixed `normalized` values are not supported")
        if len(marks) > 1:
            clash = _overlapping_added_tokens([a["content"] for a in j["added_tokens"] if a.get("normalized")],
                                              [a["content"] for a in j["added_tokens"] if not a.get("normalized")])
            if clash:
                raise ValueError(f"tokenizer.json: added tokens {clash[0]!r} and {clash[1]!r} have different `normalized` values and can "
                                 "overlap in a text; `tokenizers` then matches them in two passes, which the GPU path does not implement")
        # With a normalizer, added tokens marked normalized are matched on the normalized text — a second pass the GPU path does not
        # implement.  Those marked normalized = false are cut from the raw text first, which is what the GPU path does.
        if normalizer and any(a.get("normalized", False) for a in j.get("added_tokens", [])):
            raise ValueError("tokenizer.json: added tokens with normalized = true are not supported together with a normalizer")
        strs = (C.c_char_p * max(len(added), 1))(*[k.encode() for k, _ in added]) if added else None
        return strs, _u32([v for _, v in added]), len(added)

    def _load_sentencepiece(self, j, mdl, sp):
        if mdl.get("type") != "BPE" or mdl.get("byte_fallback") is not True or mdl.get("dropout") is not None or mdl.get("ignore_merges") or \
                mdl.get("continuing_subword_prefix") is not None or mdl.get("end_of_word_suffix") is not None:
            raise ValueError("tokenizer.json: a SentencePiece-style model must be BPE with byte_fallback = true, ignore_merges = false and "
                             "no dropout / continuing_subword_prefix / end_of_word_suffix")
        vocab = mdl["vocab"]
        missing = [t for t in [f"<0x{b:02X}>" for b in range(256)] + [METASPACE] if t not in vocab]
        if missing:
            raise ValueError(f"tokenizer.json: the vocabulary lacks {missing[0]!r} (byte fallback needs <0x00> … <0xFF>, and ▁ must be a token)")
        toks = [s.encode("utf-8") for s in vocab]   # raw UTF-8: no byte-level mapping
        merges = []
        for m in mdl.get("merges", []):
            a, b = m.split(" ") if isinstance(m, str) else m
            merges += [vocab[a], vocab[b]]
        offs = np.zeros(len(toks) + 1, dtype=np.uint32)
        np.cumsum([len(t) for t in toks], out=offs[1:])
        blob = np.frombuffer(b"".join(toks), dtype=np.uint8).copy()
        strs, sp_ids, n_added = self._added_tokens(j, sp[0] == _lib.SP_LEGACY)
        self.growth = 2   # a stretch of L bytes has at most L + 1 initial symbols
        ids, mg = _u32(list(vocab.values())), _u32(merges)
        try:
            self.h.call("smgx_tokenizer_load_bpe_metaspace", self.model, _p(blob), _p(offs), _p(ids), len(toks), _p(mg), len(merges) // 2,
                        strs, _p(sp_ids), n_added, *sp)
        except _lib.SmgxError as e:
            if e.code != _lib.TOKENIZATION_ERROR:
                raise
            raise ValueError(f"tokenizer.json: {e}") from e


TREE_BATCH_MODES = {"sequential": 0, "snapshot": 1}   # smgx_tree_batch_mode (include/smgx.h)


class CacheAwarePolicy:
    """policies::CacheAwarePolicy on the GPU.  select_worker keeps the reference signature; select_worker_batch is the
    batched form the host batcher uses (all requests see one fleet snapshot)."""

    def __init__(self, config: Optional[CacheAwareConfig] = None, device_id: int = 0, max_batch: int = 0, max_tokens_per_request: int = 0,
                 tree_batch_mode: str = "sequential"):
        self.config = config or CacheAwareConfig()
        self._h = _Handle(self.config, device_id, max_batch, max_tokens_per_request, TREE_BATCH_MODES[tree_batch_mode])
        self._slices = {}   # model → tuple(urls) currently registered
        self._tok_growth = {}   # model → most tokens per byte of text of its tokenizer (3 with a normalizer)
        self._monitor = None

    @classmethod
    def with_config(cls, config: CacheAwareConfig, **kw):
        return cls(config, **kw)

    def close(self):
        self._h.close()

    # -- LoadBalancingPolicy ------------------------------------------------------------------------------------
    def name(self) -> str:
        return _lib.load().smgx_policy_name().decode()

    def needs_request_text(self) -> bool:  # cache_aware.rs:708-710
        return True

    def on_request_complete(self, worker_url: str, success: bool):  # cache_aware.rs:692-702 (no state)
        return None

    # -- fleet ---------------------------------------------------------------------------------------------------
    def _model_of(self, workers: Sequence[BasicWorker]) -> str:
        for w in workers:  # model of the first healthy worker (cache_aware.rs:659); any worker when none is healthy
            if w.is_healthy() and w.circuit_breaker_can_execute():
                return normalize_model_key(w.model_id())
        return normalize_model_key(workers[0].model_id()) if workers else UNKNOWN_MODEL_ID

    def _register(self, model: str, urls):
        arr = (C.c_char_p * len(urls))(*[u.encode() for u in urls])
        self._h.call("smgx_set_workers", model.encode(), arr, len(urls))
        self._slices[model] = tuple(urls)

    def init_workers(self, workers: Sequence[BasicWorker]):  # cache_aware.rs:219-249
        by_model = {}
        for w in workers:
            by_model.setdefault(normalize_model_key(w.model_id()), []).append(w.url())
        for model, urls in by_model.items():
            self._register(model, urls)

    def add_worker(self, worker: BasicWorker):  # cache_aware.rs:252-266
        self._h.call("smgx_add_worker", normalize_model_key(worker.model_id()).encode(), worker.url().encode())

    def remove_worker_by_url(self, url: str):  # cache_aware.rs:302-308 (no-op)
        self._h.call("smgx_remove_worker", b"", url.encode())

    def _push_fleet(self, workers: Sequence[BasicWorker]) -> bytes:
        model = self._model_of(workers)
        urls = tuple(w.url() for w in workers)
        if self._slices.get(model) != urls:
            self._register(model, list(urls))
        loads = _u64([w.load() for w in workers])
        healthy = np.ascontiguousarray(np.asarray([1 if w.is_healthy() else 0 for w in workers], dtype=np.uint8))
        circuit = np.ascontiguousarray(np.asarray([1 if w.circuit_breaker_can_execute() else 0 for w in workers], dtype=np.uint8))
        self._h.call("smgx_set_fleet_state", model.encode(), _p(loads), _p(healthy), _p(circuit), len(workers))
        return model.encode()

    # -- KV events -----------------------------------------------------------------------------------------------
    def kv_event_monitor(self, default_block_size: Optional[int] = None) -> KvEventMonitor:
        return KvEventMonitor(self, default_block_size)

    def set_kv_event_monitor(self, monitor: Optional[KvEventMonitor]):  # cache_aware.rs:213-215
        self._monitor = monitor
        self._h.call("smgx_set_kv_event_monitor", 1 if monitor is not None else 0)

    # -- the pick ------------------------------------------------------------------------------------------------
    def select_worker(self, workers: Sequence[BasicWorker], info: SelectWorkerInfo) -> Optional[int]:
        """LoadBalancingPolicy::select_worker (cache_aware.rs:648): index into `workers` or None."""
        if not workers:
            return None
        if info.tokens is None:   # HTTP routers: string tree on request_text.unwrap_or("") (cache_aware.rs:688-689)
            idx, _ = self.select_worker_batch_request_text(workers, [info.request_text or ""])
        else:
            idx, _ = self.select_worker_batch(workers, [info.tokens])
        i = int(idx[0])
        if i >= 0:
            workers[i]._processed += 1  # mirror of increment_processed(); the library keeps the authoritative counters
        return None if i < 0 else i

    def select_worker_batch(self, workers: Sequence[BasicWorker], requests=None, tokens=None, offsets=None, want_info: bool = True):
        """Batch of token requests against one fleet snapshot.  Either `requests` (list of token lists) or a ragged
        (tokens u32, offsets u32[n+1]) pair.  → (worker_idx int32[n] with -1 = None, info structured array or None)."""
        model = self._push_fleet(workers)
        if requests is not None:
            lens = [len(r) for r in requests]
            offsets = np.zeros(len(requests) + 1, dtype=np.uint32)
            np.cumsum(lens, out=offsets[1:])
            tokens = _u32(np.concatenate([np.asarray(r, dtype=np.uint32) for r in requests]) if sum(lens) else [])
        tokens, offsets = _u32(tokens), _u32(offsets)
        n = offsets.size - 1
        out = np.full(max(n, 1), -1, dtype=np.int32)
        info = (_lib.DecisionInfo * max(n, 1))() if want_info else None
        tok_ptr = _p(tokens) if tokens.size else C.cast(C.create_string_buffer(4), C.c_void_p)
        self._h.call("smgx_select_batch_tokens", model, tok_ptr, _p(offsets), n, _p(out), C.cast(info, C.c_void_p) if info is not None else None)
        return out[:n], (info if info is None else [info[i] for i in range(n)])

    def select_worker_batch_request_text(self, workers: Sequence[BasicWorker], texts=None, want_info: bool = True, data=None, offsets=None):
        """Batch of HTTP-mode requests (request_text, no tokens) against one fleet snapshot: string-tree walk + pick on the
        GPU (select_worker_with_text, cache_aware.rs:907-974).  Either `texts` (list of str) or a ragged UTF-8 pair
        (data uint8, offsets uint32[n+1]).  → (worker_idx int32[n], info list with char counts)."""
        model = self._push_fleet(workers)
        if texts is not None:
            data, offsets = TiktokenTokenizer._ragged(texts)
        n = offsets.size - 1
        out = np.full(max(n, 1), -1, dtype=np.int32)
        info = (_lib.DecisionInfo * max(n, 1))() if want_info else None
        self._h.call("smgx_select_batch_request_text", model, _p(data), _p(offsets), n, _p(out), C.cast(info, C.c_void_p) if info is not None else None)
        return out[:n], (info if info is None else [info[i] for i in range(n)])

    # -- mesh path hashes / hash_index (crates/mesh/src/hash.rs; cache_aware.rs:95-101) ---------------------------------
    def hash_token_paths(self, requests):
        lens = [len(r) for r in requests]
        offsets = np.zeros(len(requests) + 1, dtype=np.uint32)
        np.cumsum(lens, out=offsets[1:])
        tokens = _u32(np.concatenate([np.asarray(r, dtype=np.uint32) for r in requests]) if sum(lens) else [])
        out = np.zeros(max(len(requests), 1), np.uint64)
        self._h.call("smgx_hash_token_paths", _p(tokens), _p(offsets), len(requests), _p(out))
        return out[:len(requests)]

    def hash_node_paths(self, texts):
        data, offsets = TiktokenTokenizer._ragged(texts)
        out = np.zeros(max(len(texts), 1), np.uint64)
        self._h.call("smgx_hash_node_paths", _p(data), _p(offsets), len(texts), _p(out))
        return out[:len(texts)]

    def hash_index_size(self, kind: str = "tokens", model: str = UNKNOWN_MODEL_ID) -> int:
        out = C.c_uint64()
        self._h.call("smgx_hash_index_size", model.encode(), 1 if kind == "text" else 0, C.byref(out))
        return out.value

    def hash_index_get(self, path_hash: int, kind: str = "tokens", model: str = UNKNOWN_MODEL_ID):
        """hash_index[model].token_tree / .string_tree lookup → matched-prefix copy (list of ids / str) or None."""
        nb, found = C.c_uint32(), C.c_int()
        tk = 1 if kind == "text" else 0
        self._h.call("smgx_hash_index_get", model.encode(), tk, int(path_hash), None, 0, C.byref(nb), C.byref(found))
        if not found.value:
            return None
        buf = np.zeros(max(nb.value, 1), np.uint8)
        self._h.call("smgx_hash_index_get", model.encode(), tk, int(path_hash), _p(buf), nb.value, C.byref(nb), C.byref(found))
        raw = buf[:nb.value].tobytes()
        return raw.decode("utf-8") if tk else np.frombuffer(raw, dtype=np.uint32).tolist()

    # -- TreeHandle (cache_aware.rs:454-645) ----------------------------------------------------------------------------
    def apply_known_remote_insert(self, model_id: str, tree_kind: str, node_hash: int, worker_url: str) -> bool:
        known = C.c_int()
        self._h.call("smgx_tree_apply_known_remote_insert", (model_id or "").encode(), 1 if tree_kind == "token" else 0, int(node_hash), worker_url.encode(), C.byref(known))
        return bool(known.value)

    def apply_repair_page(self, model_id: str, tree_kind: str, entries) -> int:
        """entries: [("string", path: str, [(tenant, epoch)]) | ("token", tokens, [(tenant, epoch)])] → entries applied."""
        arr = (_lib.RepairEntry * max(len(entries), 1))()
        keep = []
        for i, (kind, path, tenants) in enumerate(entries):
            data = np.frombuffer(path.encode(), dtype=np.uint8).copy() if kind == "string" else _u32(path)
            names = (C.c_char_p * max(len(tenants), 1))(*[t.encode() for t, _ in tenants])
            keep.append((data, names))
            arr[i].kind = 1 if kind == "token" else 0
            arr[i].len = data.size
            arr[i].data = data.ctypes.data if data.size else None
            arr[i].tenants = names
            arr[i].n_tenants = len(tenants)
        applied = C.c_uint32()
        self._h.call("smgx_tree_apply_repair_page", (model_id or "").encode(), 1 if tree_kind == "token" else 0, C.cast(arr, C.c_void_p), len(entries), C.byref(applied))
        return applied.value

    def set_load_feedback(self, enabled: bool):
        """Event-driven batches as a request STREAM: every pick bumps its worker's load before the next request is decided
        (WorkerLoadGuard, routers/http/router.rs:319-321); off = one frozen fleet snapshot per batch."""
        self._h.call("smgx_set_load_feedback", 1 if enabled else 0)

    def set_load_feedback_all_modes(self, enabled: bool):
        """Every cache_aware mode as a request STREAM (SMGX_FEEDBACK_CACHE_AWARE): the event-driven calls as set_load_feedback(True) does,
        and the token-tree and string-tree calls, whose imbalance gate, min-load picks and healthy[0] fallback then read the snapshot loads
        plus one per earlier pick of the call.  Refused in the "snapshot" tree batch mode.  This and set_load_feedback set one state: the
        last call wins."""
        self._h.call("smgx_set_load_feedback_policies", 1 if enabled else 0)

    def set_tree_batch_mode(self, mode: str):
        self._h.call("smgx_set_tree_batch_mode", TREE_BATCH_MODES[mode])

    # -- tokenizer + text-in pick (the whole hot path on the device) ------------------------------------------------
    def load_tiktoken_tokenizer(self, path: str, special_tokens=None, model: str = UNKNOWN_MODEL_ID, encoding: str = "cl100k_base") -> TiktokenTokenizer:
        tok = TiktokenTokenizer(self._h, model, path, special_tokens, encoding)
        self._tok_growth[normalize_model_key(model)] = tok.growth
        return tok

    def load_hf_tokenizer(self, path: str, model: str = UNKNOWN_MODEL_ID) -> HuggingFaceTokenizer:
        tok = HuggingFaceTokenizer(self._h, model, path)
        self._tok_growth[normalize_model_key(model)] = tok.growth
        return tok

    def select_worker_batch_text(self, workers: Sequence[BasicWorker], texts, want_tokens: bool = True):
        """Chat-template-rendered texts → (worker_idx, info, token lists): tokenise on the GPU, then the cache-aware pick,
        without the tokens visiting the host in between (preparation.rs:134 + worker_selection.rs:157 in one call)."""
        model = self._push_fleet(workers)
        data, offsets = TiktokenTokenizer._ragged(texts)
        n = len(texts)
        out = np.full(max(n, 1), -1, dtype=np.int32)
        info = (_lib.DecisionInfo * max(n, 1))()
        cap = self._tok_growth.get(model.decode(), 1) * int(offsets[-1]) + 1
        toks, toff = (np.zeros(cap, np.uint32), np.zeros(n + 1, np.uint32)) if want_tokens else (None, None)
        self._h.call("smgx_select_batch_text", model, _p(data), _p(offsets), n, _p(out), C.cast(info, C.c_void_p),
                     _p(toks) if want_tokens else None, _p(toff) if want_tokens else None, cap)
        tokens = [toks[toff[i]:toff[i + 1]].tolist() for i in range(n)] if want_tokens else None
        return out[:n], [info[i] for i in range(n)], tokens

    def evict_cache(self, max_size: int):  # cache_aware.rs:311-352
        self._h.call("smgx_evict_cache", max_size)

    def token_tree(self, model: str = UNKNOWN_MODEL_ID) -> TokenTree:
        t = TokenTree.__new__(TokenTree)
        t.h, t.model = self._h, model.encode()
        return t

    def string_tree(self, model: str = UNKNOWN_MODEL_ID) -> "Tree":
        return Tree(self._h, model)

    def take_processed(self, model: str = UNKNOWN_MODEL_ID, n: Optional[int] = None):
        n = n if n is not None else len(self._slices.get(model, ()))
        out = np.zeros(max(n, 1), dtype=np.uint64)
        self._h.call("smgx_take_processed", model.encode(), _p(out), n)
        return out[:n]

    def kernel_launches(self) -> int:
        return _lib.load().smgx_kernel_launches(self._h.p)


# ---- adjacent policy on the same plumbing: prefix_hash (SURVEY §8f rank 4) ---------------------------------------------------------
PREFIX_BRANCHES = ["no_healthy_workers", "no_tokens", "ring_hit", "load_balance_walk", "fallback_least_load"]   # prefix_hash.rs:70-83


@dataclass
class PrefixHashConfig:  # policies/prefix_hash.rs:38-58
    prefix_token_count: int = 256
    load_factor: float = 1.25


class HashRing:
    """worker::HashRing (model_gateway/src/worker/hash_ring.rs): 150 virtual nodes per URL at blake3("{url}#{vnode}")[..8], hashed on
    the GPU and kept sorted inside the library.  Bound to (policy handle, model) like the registry's per-model ring."""
    _seq = 0

    def __init__(self, urls, handle: Optional[_Handle] = None, model: Optional[str] = None, device_id: int = 0):
        self._h = handle or _Handle(CacheAwareConfig(eviction_interval_secs=0), device_id)
        if model is None:
            HashRing._seq += 1
            model = f"__ring_{HashRing._seq}"
        self.model = normalize_model_key(model).encode()
        self.urls = [str(u) for u in urls]
        enc = [u.encode() for u in self.urls]
        arr = (C.c_char_p * max(len(enc), 1))(*enc)
        self._h.call("smgx_hash_ring_set", self.model, arr, len(enc))

    def entries(self):
        n = C.c_uint32(0)
        self._h.call("smgx_hash_ring_entries", self.model, None, None, 0, C.byref(n))
        pos, url = np.zeros(max(n.value, 1), np.uint64), np.zeros(max(n.value, 1), np.uint32)
        self._h.call("smgx_hash_ring_entries", self.model, _p(pos), _p(url), n.value, C.byref(n))
        return pos[:n.value], url[:n.value]

    def __len__(self):  # HashRing::len (:142-144)
        n = C.c_uint32(0)
        self._h.call("smgx_hash_ring_entries", self.model, None, None, 0, C.byref(n))
        return n.value

    def is_empty(self):
        return len(self) == 0

    def worker_count(self):  # :147-149
        return len(self) // 150

    def find_healthy_urls(self, keys, is_healthy):
        """find_healthy_url (:102-134) for a batch of keys on the GPU → list of URL or None."""
        data, offsets = TiktokenTokenizer._ragged(list(keys))
        ok = np.ascontiguousarray(np.asarray([1 if is_healthy(u) else 0 for u in self.urls] or [0], dtype=np.uint8))
        n = offsets.size - 1
        out = np.full(max(n, 1), -1, np.int32)
        self._h.call("smgx_hash_ring_find_healthy", self.model, _p(data), _p(offsets), n, _p(ok), _p(out))
        return [None if i < 0 else self.urls[i] for i in out[:n]]

    def find_healthy_url(self, key: str, is_healthy):
        return self.find_healthy_urls([key], is_healthy)[0]


def _push_ring_fleet(policy, workers, ring: Optional[HashRing], with_circuit: bool) -> bytes:
    """The slice, loads and is_healthy() of a ring-reading policy (policy._h, _slices, _ring_of), plus the circuit-breaker bits when asked,
    in one smgx_set_fleet_state call.  The ring is per model in the reference (SelectWorkerInfo.hash_ring comes from the registry keyed by
    model id); a call without a ring uses the model's own state with the ring cleared."""
    model = ring.model if ring is not None else normalize_model_key(workers[0].model_id() if workers else "").encode()
    if ring is not None and ring._h is not policy._h:
        raise ValueError(f"hash ring belongs to another policy handle: build it with {type(policy).__name__}.hash_ring()")
    if ring is None and model in policy._ring_of:
        policy._h.call("smgx_hash_ring_clear", model)
        del policy._ring_of[model]
    urls = tuple(w.url() for w in workers)
    if policy._slices.get(model) != urls:
        enc = [u.encode() for u in urls]
        arr = (C.c_char_p * max(len(enc), 1))(*enc)
        policy._h.call("smgx_set_workers", model, arr, len(enc))
        policy._slices[model] = urls
    loads = _u64([w.load() for w in workers])
    healthy = np.ascontiguousarray(np.asarray([1 if w.is_healthy() else 0 for w in workers] or [0], dtype=np.uint8))
    circuit = None
    if with_circuit:
        circuit = np.ascontiguousarray(np.asarray([1 if w.circuit_breaker_can_execute() else 0 for w in workers] or [0], dtype=np.uint8))
    policy._h.call("smgx_set_fleet_state", model, _p(loads) if len(workers) else None, _p(healthy), _p(circuit) if with_circuit else None, len(workers))
    return model


def _bind_ring(policy, urls, model: str) -> HashRing:
    """The registry's per-model ring (worker/registry.rs get_hash_ring), bound to the policy's device state."""
    ring = HashRing(urls, handle=policy._h, model=model)
    policy._ring_of[ring.model] = ring
    return ring


def _seed_sequence(seed: int, call: int) -> int:
    """The seed of a policy's call-th batch, for the policies whose reference draws from rand::rng()."""
    return (seed + 0xD1B54A32D192ED03 * call) & (2**64 - 1)


class PrefixHashPolicy:
    """policies::PrefixHashPolicy (prefix_hash.rs:87-235) on the GPU: XXH3 of the first N tokens → ring lookup → bounded-load check."""

    def __init__(self, config: Optional[PrefixHashConfig] = None, device_id: int = 0, max_batch: int = 0):
        self.config = config or PrefixHashConfig()
        self._h = _Handle(CacheAwareConfig(eviction_interval_secs=0), device_id, max_batch)
        self._h.call("smgx_prefix_hash_configure", int(self.config.prefix_token_count), float(self.config.load_factor))
        self._slices = {}
        self._ring_of = {}

    def set_load_feedback(self, enabled: bool):
        """Batches as the request stream of a router that guards every pick (the gRPC router, routers/grpc/context.rs:248-259): request i
        sees the snapshot loads plus one per pick of requests < i, in the bound (Σ load + 1) / n × load_factor and the least loaded fallback.
        Every batch of one device-resident call forms one stream.  Off = one frozen fleet snapshot per batch."""
        self._h.call("smgx_set_load_feedback_policies", 2 if enabled else 0)

    @classmethod
    def with_defaults(cls, **kw):  # :100-103
        return cls(PrefixHashConfig(), **kw)

    def name(self) -> str:  # :231-233
        return "prefix_hash"

    def needs_request_text(self) -> bool:  # trait default (policies/mod.rs:77-79)
        return False

    def on_request_complete(self, worker_url: str, success: bool):  # trait default: no state
        return None

    def hash_ring(self, urls, model: str = UNKNOWN_MODEL_ID) -> HashRing:
        """The registry's per-model ring (worker/registry.rs get_hash_ring), bound to this policy's device state."""
        return _bind_ring(self, urls, model)

    def compute_prefix_hashes(self, requests):  # compute_prefix_hash (:106-113) for a batch
        tokens, offsets = _ragged_tokens(requests)
        n = offsets.size - 1
        out = np.zeros(max(n, 1), np.uint64)
        self._h.call("smgx_prefix_hashes", _tok_ptr(tokens), _p(offsets), n, _p(out))
        return out[:n]

    def _push_fleet(self, workers, ring: Optional[HashRing]) -> bytes:
        return _push_ring_fleet(self, workers, ring, with_circuit=False)

    def select_worker_batch(self, workers, requests=None, ring: Optional[HashRing] = None, tokens=None, offsets=None, has_tokens=None):
        """One batch against one fleet snapshot → (idx int32[n] with -1 = None, branch names)."""
        model = self._push_fleet(workers, ring)
        if requests is not None:
            has_tokens = [0 if r is None else 1 for r in requests]
            tokens, offsets = _ragged_tokens([[] if r is None else r for r in requests])
            if all(has_tokens):
                has_tokens = None
        tokens, offsets = _u32(tokens), _u32(offsets)
        n = offsets.size - 1
        out = np.full(max(n, 1), -1, np.int32)
        info = (_lib.DecisionInfo * max(n, 1))()
        flags = None if has_tokens is None else np.ascontiguousarray(np.asarray(has_tokens, np.uint8))
        self._h.call("smgx_prefix_hash_select_batch_tokens", model, _tok_ptr(tokens), _p(offsets), n, _p(flags) if flags is not None else None, _p(out),
                     C.cast(info, C.c_void_p))
        return out[:n], [PREFIX_BRANCHES[info[i].branch] for i in range(n)]

    def select_worker_impl(self, workers, info: SelectWorkerInfo):  # :203-222 → (Option<usize>, Branch)
        idx, br = self.select_worker_batch(workers, [info.tokens], ring=info.hash_ring)
        return (None if idx[0] < 0 else int(idx[0])), br[0]

    def select_worker(self, workers, info: SelectWorkerInfo) -> Optional[int]:  # LoadBalancingPolicy::select_worker (:225-229)
        return self.select_worker_impl(workers, info)[0]

    def kernel_launches(self) -> int:
        return int(self._h.L.smgx_kernel_launches(self._h.p))


def _ragged_tokens(requests):
    lens = [len(r) for r in requests]
    offsets = np.zeros(len(requests) + 1, dtype=np.uint32)
    np.cumsum(lens, out=offsets[1:])
    tokens = _u32(np.concatenate([np.asarray(r, dtype=np.uint32) for r in requests]) if sum(lens) else [])
    return tokens, offsets


def _tok_ptr(tokens):
    return _p(tokens) if tokens.size else C.cast(C.create_string_buffer(4), C.c_void_p)


class PowerOfTwoPolicy:
    """policies::PowerOfTwoPolicy (power_of_two.rs:18-135) on the GPU: two random healthy candidates per request, the less loaded one wins
    (token usage when both have a cached load response, request counts otherwise).  The reference draws from a thread-local generator;
    here every call consumes one value of a per-policy seed sequence and request i of the call uses draws 2i, 2i + 1 of that stream."""

    def __init__(self, device_id: int = 0, max_batch: int = 0, seed: int = 0x5EED):
        self._h = _Handle(CacheAwareConfig(eviction_interval_secs=0), device_id, max_batch)
        self._slices = {}
        self._seed = int(seed) & (2**64 - 1)
        self._calls = 0

    def name(self) -> str:  # :122-124
        return "power_of_two"

    def needs_request_text(self) -> bool:  # trait default (policies/mod.rs:77-79)
        return False

    def update_loads(self, loads: dict):
        """update_loads (:129-135): url → WorkerLoadResponse; a value may be the response's per-DP-rank token_usage list (→ its mean,
        effective_token_usage, protocols worker.rs:1039-1044, 0.0 when empty) or that number itself."""
        if not loads:
            return
        urls = [u.encode() for u in loads]
        vals = []
        for v in loads.values():
            if isinstance(v, (list, tuple, np.ndarray)):
                vals.append(float(np.sum(np.asarray(v, np.float64)) / len(v)) if len(v) else 0.0)
            else:
                vals.append(float(v))
        arr = (C.c_char_p * len(urls))(*urls)
        usage = np.ascontiguousarray(np.asarray(vals, np.float64))
        self._h.call("smgx_power_of_two_update_loads", arr, _p(usage), len(urls))

    def _push_fleet(self, workers) -> bytes:
        model = normalize_model_key(workers[0].model_id() if workers else "").encode()
        urls = tuple(w.url() for w in workers)
        if self._slices.get(model) != urls:
            enc = [u.encode() for u in urls]
            arr = (C.c_char_p * max(len(enc), 1))(*enc)
            self._h.call("smgx_set_workers", model, arr, len(enc))
            self._slices[model] = urls
        loads = _u64([w.load() for w in workers])
        healthy = np.ascontiguousarray(np.asarray([1 if w.is_healthy() else 0 for w in workers] or [0], dtype=np.uint8))
        circuit = np.ascontiguousarray(np.asarray([1 if w.circuit_breaker_can_execute() else 0 for w in workers] or [0], dtype=np.uint8))
        self._h.call("smgx_set_fleet_state", model, _p(loads) if len(workers) else None, _p(healthy), _p(circuit), len(workers))
        return model

    def set_load_feedback(self, enabled: bool):
        """Batches as the request stream of a router that guards every pick (the gRPC router, routers/grpc/context.rs:248-259): the draws
        and pairs are unchanged, the request-count comparison reads the snapshot loads plus one per pick of requests < i."""
        self._h.call("smgx_set_load_feedback_policies", 4 if enabled else 0)

    def next_seed(self) -> int:
        self._calls += 1
        return _seed_sequence(self._seed, self._calls)

    def select_worker_batch(self, workers, n: int, seed: Optional[int] = None, with_details: bool = False):
        """n requests against one fleet snapshot → idx int32[n] (-1 = None) [, pairs int32[n, 2], metric uint8[n]]."""
        model = self._push_fleet(workers)
        seed = self.next_seed() if seed is None else int(seed) & (2**64 - 1)
        out = np.full(max(n, 1), -1, np.int32)
        pairs = np.full((max(n, 1), 2), -1, np.int32)
        metric = np.zeros(max(n, 1), np.uint8)
        self._h.call("smgx_power_of_two_select_batch", model, n, seed, _p(out), _p(pairs), _p(metric) if with_details else None)
        for i, pr in zip(out[:n], pairs[:n]):
            if i >= 0 and pr[0] >= 0 and hasattr(workers[int(i)], "increment_processed"):
                workers[int(i)].increment_processed()        # :110 (not on the single-healthy-worker early return, :44-46)
        return (out[:n], pairs[:n], metric[:n]) if with_details else out[:n]

    def select_worker(self, workers, info=None) -> Optional[int]:
        """LoadBalancingPolicy::select_worker (:36-120)."""
        if not workers:
            return None
        idx = self.select_worker_batch(workers, 1)
        return None if idx[0] < 0 else int(idx[0])


# ---- adjacent policy on the same plumbing: consistent_hashing ----------------------------------------------------------------------
CH_HEADERS = ("x-smg-target-worker", "x-smg-routing-key", "authorization", "x-forwarded-for", "cookie")
CH_BRANCHES = ["no_healthy_workers", "target_worker_hit", "target_worker_miss", "routing_key_hit", "random_fallback"]   # Branch::as_str


def _ch_header_values(headers):
    """The five values HeaderMap::get returns for CH_HEADERS (None = absent); names are case-insensitive, a repeated header (a list
    value, or the same name twice in an item list) yields its first value."""
    vals = [None] * len(CH_HEADERS)
    if headers is None:
        return vals
    for name, v in (headers.items() if hasattr(headers, "items") else headers):
        name = name.decode() if isinstance(name, (bytes, bytearray)) else str(name)
        try:
            h = CH_HEADERS.index(name.lower())
        except ValueError:
            continue
        if isinstance(v, (list, tuple)):
            if not v:
                continue
            v = v[0]
        if vals[h] is None:
            vals[h] = v.encode("utf-8") if isinstance(v, str) else bytes(v)
    return vals


class ConsistentHashingPolicy:
    """policies::ConsistentHashingPolicy (consistent_hashing.rs) on the GPU: X-SMG-Target-Worker, then X-SMG-Routing-Key, then the first
    present of authorization / x-forwarded-for / cookie hashed onto the ring (or modulo the healthy URLs without a ring), else a random
    healthy worker.  The reference draws that worker from a thread-local generator; here every call consumes one value of a per-policy
    seed sequence and request i of the call uses draw i of that stream."""

    def __init__(self, device_id: int = 0, max_batch: int = 0, seed: int = 0x5EED):
        self._h = _Handle(CacheAwareConfig(eviction_interval_secs=0), device_id, max_batch)
        self._slices = {}
        self._ring_of = {}
        self._seed = int(seed) & (2**64 - 1)
        self._calls = 0

    def hash_ring(self, urls, model: str = UNKNOWN_MODEL_ID) -> HashRing:
        """The registry's per-model ring (worker/registry.rs get_hash_ring), bound to this policy's device state."""
        return _bind_ring(self, urls, model)

    def next_seed(self) -> int:
        self._calls += 1
        return _seed_sequence(self._seed, self._calls)

    def _push_fleet(self, workers, ring: Optional[HashRing]) -> bytes:
        # the circuit-breaker bits go with the fleet although no pick reads them, so the device sees the fleet the router has
        return _push_ring_fleet(self, workers, ring, with_circuit=True)

    def name(self) -> str:  # :188-190
        return "consistent_hashing"

    def needs_request_text(self) -> bool:  # trait default (policies/mod.rs:77-79)
        return False

    def on_request_complete(self, worker_url: str, success: bool):  # trait default: no state
        return None

    def select_worker_batch(self, workers, headers_list=None, ring: Optional[HashRing] = None, seed: Optional[int] = None, with_details: bool = False,
                            values=None, offsets=None, present=None):
        """One batch against one fleet snapshot → idx int32[n] (-1 = None) [, branch names, key positions uint64[n]].  headers_list[i] is
        request i's headers (a mapping, an item list, or None for info.headers = None); or pass the packed form of the C call directly:
        values (bytes), offsets (5n + 1), present (n bit masks)."""
        model = self._push_fleet(workers, ring)
        seed = self.next_seed() if seed is None else int(seed) & (2**64 - 1)
        if headers_list is not None:
            blob, offs, present = bytearray(), [0], []
            for hd in headers_list:
                bits = 0
                for h, v in enumerate(_ch_header_values(hd)):
                    if v is not None:
                        bits |= 1 << h
                        blob += v
                    offs.append(len(blob))
                present.append(bits)
            values, offsets = bytes(blob), offs
        offsets = _u32(offsets)
        present = np.ascontiguousarray(np.asarray(present, np.uint8))
        n = present.size
        if offsets.size != len(CH_HEADERS) * n + 1:
            raise ValueError("offsets must hold 5 n + 1 entries")
        vbuf = np.frombuffer(values, np.uint8) if values else np.zeros(0, np.uint8)
        out = np.full(max(n, 1), -1, np.int32)
        branch = np.zeros(max(n, 1), np.uint8)
        key_pos = np.zeros(max(n, 1), np.uint64)
        self._h.call("smgx_consistent_hashing_select_batch", model, n, _p(vbuf), _p(offsets), _p(present), seed, _p(out),
                     _p(branch) if with_details else None, _p(key_pos) if with_details else None)
        if with_details:
            return out[:n], [CH_BRANCHES[b] for b in branch[:n]], key_pos[:n]
        return out[:n]

    def select_worker_impl(self, workers, info: SelectWorkerInfo):  # :116-186 → (Option<usize>, Branch)
        idx, br, _ = self.select_worker_batch(workers, [info.headers], ring=info.hash_ring, with_details=True)
        return (None if idx[0] < 0 else int(idx[0])), br[0]

    def select_worker(self, workers, info: Optional[SelectWorkerInfo] = None) -> Optional[int]:  # LoadBalancingPolicy::select_worker (:182-186)
        return self.select_worker_impl(workers, info or SelectWorkerInfo())[0]

    def kernel_launches(self) -> int:
        return int(self._h.L.smgx_kernel_launches(self._h.p))


class PolicyFactory:
    """policies::PolicyFactory for the one policy this library replaces (factory.rs:17-93)."""

    @staticmethod
    def create_by_name(name: str, **kw):
        if name.lower() in ("cache_aware", "cacheaware"):  # factory.rs:84
            return CacheAwarePolicy(CacheAwareConfig(), **kw)
        if name.lower() in ("prefix_hash", "prefixhash"):  # factory.rs:90
            return PrefixHashPolicy.with_defaults(**kw)
        if name.lower() in ("power_of_two", "poweroftwo"):  # factory.rs:83
            return PowerOfTwoPolicy(**kw)
        if name.lower() in ("consistent_hashing", "consistenthashing"):  # factory.rs:87
            return ConsistentHashingPolicy(**kw)
        return None

    @staticmethod
    def create_from_config(cache_threshold, balance_abs_threshold, balance_rel_threshold, eviction_interval_secs, max_tree_size, block_size,
                           **kw):  # factory.rs:22-39 PolicyConfig::CacheAware{..}
        return CacheAwarePolicy(CacheAwareConfig(cache_threshold, balance_abs_threshold, balance_rel_threshold, eviction_interval_secs,
                                                 max_tree_size, block_size), **kw)
