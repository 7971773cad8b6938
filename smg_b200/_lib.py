"""ctypes binding of the smgx C ABI (include/smgx.h).  The library is the product; this file only declares
signatures.  Loading fails loudly when libsmgx.so has not been built — there is no Python/CPU fallback."""
import ctypes as C
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsmgx.so")
HEADER = os.path.join(os.path.dirname(HERE), "include", "smgx.h")

SUCCESS, INVALID_ARGUMENT, TOKENIZATION_ERROR, MEMORY_ERROR, DEVICE_ERROR = 0, 1, 2, 4, 5
WORKER_NOT_TRACKED, PARENT_BLOCK_NOT_FOUND, NOT_FOUND, BUSY, UNKNOWN_ERROR = 10, 11, 12, 13, 99
PRETOK_CL100K, PRETOK_R50K, PRETOK_QWEN2, PRETOK_DEEPSEEK = 0, 1, 2, 4   # smgx_pretokenizer
NORMALIZER_NONE, NORMALIZER_NFC = 0, 1   # smgx_normalizer
SP_LEGACY, SP_METASPACE = 0, 1   # smgx_sp_shape
PREPEND_NEVER, PREPEND_FIRST, PREPEND_ALWAYS = 0, 1, 2   # smgx_prepend_scheme

BRANCHES = ["no_healthy", "imbalanced_min_load", "event_overlap", "event_min_load", "tree_match", "tree_min_load",
            "tree_fallback_first_healthy", "no_tree_random"]


class Config(C.Structure):
    _fields_ = [("cache_threshold", C.c_float), ("balance_abs_threshold", C.c_uint64), ("balance_rel_threshold", C.c_float),
                ("eviction_interval_secs", C.c_uint64), ("max_tree_size", C.c_uint64), ("block_size", C.c_uint64),
                ("device_id", C.c_int32), ("max_batch", C.c_uint32), ("max_tokens_per_request", C.c_uint32), ("tree_batch_mode", C.c_uint32)]


class KvEvent(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("worker_id", C.c_uint32), ("first_block", C.c_uint32), ("n_blocks", C.c_uint32),
                ("parent_block_hash", C.c_int64), ("has_parent", C.c_uint32), ("reserved", C.c_uint32)]


class RepairEntry(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("len", C.c_uint32), ("data", C.c_void_p), ("tenants", C.POINTER(C.c_char_p)), ("n_tenants", C.c_uint32), ("reserved", C.c_uint32)]


class DecisionInfo(C.Structure):
    _fields_ = [("matched", C.c_uint32), ("input", C.c_uint32), ("branch", C.c_uint8), ("nodes", C.c_uint8), ("reserved", C.c_uint8 * 2)]


class SmgxError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"smgx error {code}: {msg}")
        self.code = code
        self.msg = msg


_lib = None


def header_symbols():
    """Every function the public header declares (used by the export test)."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(smgx_[a-z0-9_]+)\s*\(", text)))


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -m smg_b200.build` (nvcc, sm_90a). "
                          "smg_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, cp, u32, u64, i64, st = C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint64, C.c_int64, C.c_int
    pp = C.POINTER(C.c_char_p)
    P = C.POINTER

    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    sig("smgx_default_config", None, P(Config))
    sig("smgx_policy_create", vp, P(Config), pp)
    sig("smgx_policy_free", None, vp)
    sig("smgx_policy_name", cp)
    sig("smgx_abi_version", u32)
    sig("smgx_free_string", None, vp)
    sig("smgx_bind_numa", st, C.c_int, P(C.c_int), pp)
    sig("smgx_alloc_pinned", vp, C.c_size_t)
    sig("smgx_free_pinned", None, vp)
    sig("smgx_set_workers", st, vp, cp, P(cp), u32, pp)
    sig("smgx_set_fleet_state", st, vp, cp, vp, vp, vp, u32, pp)
    sig("smgx_add_worker", st, vp, cp, cp, pp)
    sig("smgx_remove_worker", st, vp, cp, cp, pp)
    sig("smgx_take_processed", st, vp, cp, vp, u32, pp)
    sig("smgx_set_kv_event_monitor", st, vp, C.c_int, pp)
    sig("smgx_indexer_create", st, vp, cp, u32, pp)
    sig("smgx_indexer_set_block_size", st, vp, cp, u32, pp)
    sig("smgx_indexer_intern_worker", st, vp, cp, cp, P(u32), pp)
    sig("smgx_indexer_worker_id", st, vp, cp, cp, P(i64), pp)
    sig("smgx_indexer_apply_stored", st, vp, cp, u32, vp, vp, u32, vp, pp)
    sig("smgx_indexer_apply_stored_tokens", st, vp, cp, u32, vp, vp, u32, u32, vp, pp)
    sig("smgx_indexer_apply_removed", st, vp, cp, u32, vp, u32, pp)
    sig("smgx_indexer_apply_cleared", st, vp, cp, u32, pp)
    sig("smgx_indexer_remove_worker", st, vp, cp, u32, pp)
    sig("smgx_indexer_current_size", st, vp, cp, P(u64), pp)
    sig("smgx_indexer_entry_count", st, vp, cp, P(u64), pp)
    sig("smgx_kv_events_apply", st, vp, cp, vp, u32, vp, vp, vp, u32, P(u32), pp)
    sig("smgx_indexer_find_matches", st, vp, cp, vp, u32, C.c_int, vp, vp, u32, P(u32), pp)
    sig("smgx_content_hashes", st, vp, vp, u32, u32, vp, u32, P(u32), pp)
    sig("smgx_tree_create", st, vp, cp, C.c_int, pp)
    sig("smgx_tree_insert_tokens", st, vp, cp, vp, u32, cp, pp)
    sig("smgx_tree_insert_tokens_batch", st, vp, cp, vp, vp, u32, P(cp), pp)
    sig("smgx_tree_walk_many_device", st, vp, cp, u32, vp, vp, vp, vp, vp, pp)
    sig("smgx_tree_match_tokens", st, vp, cp, vp, u32, P(u32), P(u32), vp, u32, pp)
    sig("smgx_tree_evict_tenant", st, vp, cp, cp, u64, pp)
    sig("smgx_evict_cache", st, vp, u64, pp)
    sig("smgx_tree_tenant_size", st, vp, cp, cp, P(u64), pp)
    sig("smgx_tree_clear", st, vp, cp, pp)
    sig("smgx_tree_entries", st, vp, cp, P(C.c_void_p), pp)
    sig("smgx_hash_token_paths", st, vp, vp, vp, u32, vp, pp)
    sig("smgx_hash_node_paths", st, vp, vp, vp, u32, vp, pp)
    sig("smgx_prefix_hash_configure", st, vp, u64, C.c_double, pp)
    sig("smgx_power_of_two_update_loads", st, vp, P(cp), vp, u32, pp)
    sig("smgx_power_of_two_select_batch", st, vp, cp, u32, u64, vp, vp, vp, pp)
    sig("smgx_consistent_hashing_select_batch", st, vp, cp, u32, vp, vp, vp, u64, vp, vp, vp, pp)
    sig("smgx_hash_ring_set", st, vp, cp, P(cp), u32, pp)
    sig("smgx_hash_ring_clear", st, vp, cp, pp)
    sig("smgx_hash_ring_entries", st, vp, cp, vp, vp, u32, P(u32), pp)
    sig("smgx_hash_ring_find_healthy", st, vp, cp, vp, vp, u32, vp, vp, pp)
    sig("smgx_prefix_hashes", st, vp, vp, vp, u32, vp, pp)
    sig("smgx_prefix_hash_select_batch_tokens", st, vp, cp, vp, vp, u32, vp, vp, vp, pp)
    sig("smgx_prefix_hash_select_many_tokens_device", st, vp, cp, u32, vp, vp, vp, vp, pp)
    sig("smgx_tree_apply_known_remote_insert", st, vp, cp, C.c_int, u64, cp, P(C.c_int), pp)
    sig("smgx_tree_apply_repair_page", st, vp, cp, C.c_int, vp, u32, P(u32), pp)
    sig("smgx_hash_index_size", st, vp, cp, C.c_int, P(u64), pp)
    sig("smgx_hash_index_get", st, vp, cp, C.c_int, u64, vp, u32, P(u32), P(C.c_int), pp)
    sig("smgx_set_tree_batch_mode", st, vp, u32, pp)
    sig("smgx_stree_insert_text", st, vp, cp, vp, u32, cp, pp)
    sig("smgx_stree_match", st, vp, cp, vp, u32, P(u32), P(u32), vp, u32, pp)
    sig("smgx_stree_prefix_match_tenant", st, vp, cp, vp, u32, cp, P(u32), pp)
    sig("smgx_stree_sizes", st, vp, cp, C.c_int, P(C.c_void_p), pp)
    sig("smgx_stree_entries", st, vp, cp, P(C.c_void_p), P(u64), pp)
    sig("smgx_stree_snapshot", st, vp, cp, P(C.c_void_p), P(u64), pp)
    sig("smgx_stree_load_snapshot", st, vp, cp, vp, u64, pp)
    sig("smgx_stree_merge_snapshot", st, vp, cp, vp, u64, pp)
    sig("smgx_stree_walk_many_device", st, vp, cp, u32, vp, vp, vp, vp, vp, vp, pp)
    sig("smgx_stree_clear", st, vp, cp, pp)
    sig("smgx_stree_node_count", st, vp, cp, P(u64), pp)
    sig("smgx_select_batch_request_text", st, vp, cp, vp, vp, u32, vp, vp, pp)
    sig("smgx_tokenizer_load_tiktoken_file", st, vp, cp, cp, P(cp), vp, u32, pp)
    sig("smgx_tokenizer_load_tiktoken", st, vp, cp, vp, vp, vp, u32, P(cp), vp, u32, pp)
    sig("smgx_tokenizer_load_bpe_merges", st, vp, cp, vp, vp, vp, u32, vp, u32, C.c_int, P(cp), vp, u32, pp)
    sig("smgx_tokenizer_load_tiktoken_file_ex", st, vp, cp, cp, P(cp), vp, u32, C.c_int, pp)
    sig("smgx_tokenizer_load_tiktoken_ex", st, vp, cp, vp, vp, vp, u32, P(cp), vp, u32, C.c_int, pp)
    sig("smgx_tokenizer_load_bpe_merges_ex", st, vp, cp, vp, vp, vp, u32, vp, u32, C.c_int, P(cp), vp, u32, C.c_int, pp)
    sig("smgx_tokenizer_load_bpe_merges_norm", st, vp, cp, vp, vp, vp, u32, vp, u32, C.c_int, P(cp), vp, u32, C.c_int, C.c_int, pp)
    sig("smgx_tokenizer_load_bpe_metaspace", st, vp, cp, vp, vp, vp, u32, vp, u32, P(cp), vp, u32, C.c_int, C.c_int, C.c_int, pp)
    sig("smgx_tokenize_batch", st, vp, cp, vp, vp, u32, vp, vp, u32, pp)
    sig("smgx_select_batch_text", st, vp, cp, vp, vp, u32, vp, vp, vp, vp, u32, pp)
    sig("smgx_select_batch_tokens", st, vp, cp, vp, vp, u32, vp, vp, pp)
    sig("smgx_set_load_feedback", st, vp, C.c_int, pp)
    sig("smgx_set_load_feedback_policies", st, vp, u32, pp)
    sig("smgx_pipeline_depth", u32, vp)
    sig("smgx_submit_tokens", st, vp, cp, vp, vp, u32, vp, vp, P(u64), pp)
    sig("smgx_wait", st, vp, u64, pp)
    sig("smgx_submit_tokens_mapped", st, vp, cp, vp, vp, u32, u32, vp, vp, vp, u64, pp)
    sig("smgx_submit_text", st, vp, cp, vp, vp, u32, vp, vp, P(u64), pp)
    sig("smgx_select_batch_tokens_device", st, vp, cp, u32, vp, vp, u32, u32, vp, vp, pp)
    sig("smgx_select_many_tokens_device", st, vp, cp, u32, vp, vp, vp, u32, vp, pp)
    sig("smgx_shard_candidates_device", st, vp, cp, u32, vp, vp, u32, u32, vp, vp, pp)
    sig("smgx_shard_reduce_device", st, vp, u32, vp, vp, vp, u32, u32, vp, vp, pp)
    sig("smgx_shard_exchange_create", st, vp, u32, u32, u32, vp, pp)
    sig("smgx_shard_exchange_connect", st, vp, vp, pp)
    sig("smgx_shard_select_fused_device", st, vp, cp, u32, vp, vp, u32, u32, vp, vp, vp, pp)
    sig("smgx_device_alloc", vp, vp, C.c_size_t, pp)
    sig("smgx_device_free", None, vp, vp)
    sig("smgx_memcpy_h2d", st, vp, vp, vp, C.c_size_t, pp)
    sig("smgx_memcpy_d2h", st, vp, vp, vp, C.c_size_t, pp)
    sig("smgx_synchronize", st, vp, pp)
    sig("smgx_timer_start", st, vp, u32, pp)
    sig("smgx_timer_stop_ms", st, vp, u32, P(C.c_float), pp)
    sig("smgx_timer_start_all", st, vp, pp)
    sig("smgx_timer_start_all_gated", st, vp, u32, pp)
    sig("smgx_timer_start_gated", st, vp, u32, u32, pp)
    sig("smgx_stream_hold", st, vp, u32, u32, pp)
    sig("smgx_timer_stop_all_ms", st, vp, P(C.c_float), pp)
    sig("smgx_set_event_path", None, C.c_int, C.c_int)
    sig("smgx_set_fused_prefetch", None, C.c_int)
    sig("smgx_set_fused_tile", None, C.c_int, C.c_int64)
    sig("smgx_set_event_simple", None, C.c_int)
    sig("smgx_set_tile_depth", None, C.c_int)
    sig("smgx_kernel_launches", u64, vp)
    sig("smgx_flush_l2", st, vp, pp)
    _lib = L
    return L


def check(code, err):
    """Raise SmgxError for a non-zero status, consuming the callee-allocated message."""
    msg = ""
    if err and err.value:
        msg = err.value.decode(errors="replace")
        load().smgx_free_string(C.cast(err, C.c_void_p))
    if code != SUCCESS:
        raise SmgxError(code, msg)


def new_err():
    return C.c_char_p()
