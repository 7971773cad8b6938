/*
 * smgx — H100-native cache-aware worker pick behind a C ABI.
 *
 * Drop-in boundary for SMG's `--policy cache_aware` hot path.  The Rust side that a maintainer adds is a
 * `struct GpuCacheAwarePolicy { h: *mut smgx_policy }` implementing
 *     trait LoadBalancingPolicy            (model_gateway/src/policies/mod.rs:43-86)
 * registered at PolicyFactory::create_from_config / create_by_name
 *                                          (model_gateway/src/policies/factory.rs:22-39, :84)
 * See INTEGRATION.md for the binding.  Conventions mirror the reference's only existing C ABI
 * (bindings/golang/src/error.rs:6-15, memory.rs:10-27, tokenizer.rs:113-161):
 *   - every call returns an smgx_status (0 = success) or a nullable handle;
 *   - `char** err` is optional; on failure it receives a callee-allocated NUL-terminated message that the
 *     caller releases with smgx_free_string();
 *   - opaque handle from *_create, released by *_free; null pointer arguments → SMGX_INVALID_ARGUMENT;
 *   - hot-path buffers are CALLER-allocated (ideally pinned, see smgx_alloc_pinned); nothing is malloc'ed per call.
 *
 * There is NO CPU fallback: every select/find call runs hand-written sm_90a kernels and fails with
 * SMGX_DEVICE_ERROR when no CUDA device is usable.  No torch types, plain pointers and sizes only.
 */
#ifndef SMGX_H
#define SMGX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SMGX_ABI_VERSION 1

typedef enum smgx_status {
    SMGX_SUCCESS = 0,
    SMGX_INVALID_ARGUMENT = 1,   /* SglErrorCode::InvalidArgument  (bindings/golang/src/error.rs:9)  */
    SMGX_TOKENIZATION_ERROR = 2, /* SglErrorCode::TokenizationError                                   */
    SMGX_MEMORY_ERROR = 4,       /* SglErrorCode::MemoryError                                         */
    SMGX_DEVICE_ERROR = 5,       /* CUDA runtime / no device — there is no CPU fallback               */
    SMGX_WORKER_NOT_TRACKED = 10,    /* kv_index ApplyError::WorkerNotTracked    (event_tree.rs:90-95) */
    SMGX_PARENT_BLOCK_NOT_FOUND = 11,/* kv_index ApplyError::ParentBlockNotFound (event_tree.rs:90-95) */
    SMGX_NOT_FOUND = 12,         /* unknown model key / no indexer for the model                      */
    SMGX_BUSY = 13,              /* every pipeline lane has a submission in flight: smgx_wait one, then retry (the synchronous calls do) */
    SMGX_UNKNOWN_ERROR = 99
} smgx_status;

/* Which branch of CacheAwarePolicy::select_worker produced a pick (cache_aware.rs:648-690). */
typedef enum smgx_branch {
    SMGX_BR_NO_HEALTHY = 0,              /* healthy_indices empty → None               (:653-655) */
    SMGX_BR_IMBALANCED_MIN_LOAD = 1,     /* select_worker_min_load                     (:356-440) */
    SMGX_BR_EVENT_OVERLAP = 2,           /* score_overlap hit                          (:776-831) */
    SMGX_BR_EVENT_MIN_LOAD = 3,          /* event-driven, no overlap → min load        (:759-768) */
    SMGX_BR_TREE_MATCH = 4,              /* match_rate > cache_threshold → tenant      (:854-859) */
    SMGX_BR_TREE_MIN_LOAD = 5,           /* match_rate ≤ threshold → min load          (:860-865) */
    SMGX_BR_TREE_FALLBACK_FIRST_HEALTHY = 6, /* tenant gone/unhealthy → healthy[0]     (:892-894) */
    SMGX_BR_NO_TREE_RANDOM = 7           /* no tree for model (:896-903); smgx returns healthy[0] */
} smgx_branch;

/* CacheAwareConfig (model_gateway/src/policies/mod.rs:94-117) + device placement. */
typedef struct smgx_cache_aware_config {
    float cache_threshold;            /* default 0.5  */
    uint64_t balance_abs_threshold;   /* default 32   */
    float balance_rel_threshold;      /* default 1.1  */
    uint64_t eviction_interval_secs;  /* default 30: a background thread bounds every tree to max_tree_size at this period, as the
                                         reference does (cache_aware.rs:126-199); 0 = none (the caller drives smgx_evict_cache) */
    uint64_t max_tree_size;           /* default 10000 */
    uint64_t block_size;              /* default 16   */
    int32_t device_id;                /* CUDA ordinal; -1 = host-mirror only (index writers work, every select fails) */
    uint32_t max_batch;               /* largest n accepted by one select call (sizes device staging); 0 → 65536 */
    uint32_t max_tokens_per_request;  /* sizes per-warp scratch; 0 → 32768 */
    uint32_t tree_batch_mode;         /* smgx_tree_batch_mode; tree modes only (the event-driven mode never writes on the path) */
} smgx_cache_aware_config;

/* How a batch of tree-mode requests (token tree / string tree: every routed request also inserts) is serialised.
 * select_worker takes &self and runs on many tokio tasks at once; it is not atomic, and the reference promises eventual
 * consistency only between concurrent match and insert (token_tree.rs:1035-1037).
 *   SEQUENTIAL: results equal calling select_worker one request at a time, in batch order (timestamps included).  Run
 *               optimistically: the GPU walks the rest of the batch against one snapshot, the host commits requests in order up to
 *               the first one a preceding insert really affected, and the walk restarts there.
 *   SNAPSHOT:   every request of the batch walks and decides against the pre-batch tree (one launch), then the match side
 *               effects and the inserts are applied in batch order — the interleaving "all reads, then each task's writes" of
 *               concurrent select_worker calls.  Identical to SEQUENTIAL whenever no two requests of a batch share a first page. */
typedef enum smgx_tree_batch_mode { SMGX_TREE_BATCH_SEQUENTIAL = 0, SMGX_TREE_BATCH_SNAPSHOT = 1 } smgx_tree_batch_mode;

/* Per-request detail, optional output of the select calls. */
typedef struct smgx_decision_info {
    uint32_t matched;   /* event mode: overlap score in blocks; tree modes: matched tokens / chars */
    uint32_t input;     /* request length in tokens / chars                                        */
    uint8_t branch;     /* smgx_branch                                                             */
    uint8_t nodes;      /* tree modes: nodes the walk counted (saturates at 255); 0 in event mode  */
    uint8_t reserved[2];
} smgx_decision_info;

/* Worker-id-sharded fleets (BASELINE config 4: 4096 workers, 512 per GPU; SURVEY §8e).  Each shard holds a contiguous
 * range of the global worker slice and emits, per request, its best local candidate; the shards' candidates are exchanged
 * (all-gather, 24 B per request per shard) and merged with smgx_shard_reduce_device on every rank. */
typedef struct smgx_shard_candidate {
    uint32_t score;      /* overlap blocks of the shard's best eligible worker; 0 = no eligible overlap in this shard */
    uint32_t local_idx;  /* its index in the SHARD's slice */
    uint64_t load;       /* tie-breaks of score_overlap (cache_aware.rs:806-818) */
    uint64_t tree_size;
} smgx_shard_candidate;
typedef struct smgx_shard_fleet {   /* the select_worker prologue of one shard (cache_aware.rs:651-670) */
    int32_t min_load_idx;    /* first argmin load() over the shard's healthy workers, -1 if none */
    int32_t first_healthy;
    uint32_t n_healthy;
    uint32_t imbalanced;     /* shard-local; the merged gate is recomputed from min_load / max_load */
    uint64_t min_load, max_load;   /* over all the shard's workers; UINT64_MAX and 0 for a shard with no workers */
    uint64_t min_healthy_load;
} smgx_shard_fleet;

typedef struct smgx_policy smgx_policy;

/* ---- lifecycle ------------------------------------------------------------------------------------------ */
void smgx_default_config(smgx_cache_aware_config* cfg);                 /* CacheAwareConfig::default() (mod.rs:106-117) */
smgx_policy* smgx_policy_create(const smgx_cache_aware_config* cfg, char** err);   /* CacheAwarePolicy::with_config (cache_aware.rs:120) */
void smgx_policy_free(smgx_policy* p);
const char* smgx_policy_name(void);                                     /* "cache_aware" (cache_aware.rs:704-706) */
uint32_t smgx_abi_version(void);
void smgx_free_string(char* s);                                         /* sgl_free_string (memory.rs:10-15) */
/* Opt-in: bind the calling thread to the CPUs of the NUMA node `device_id` is attached to and prefer that node for the memory it
 * allocates next (call it before smgx_alloc_pinned / smgx_policy_create on multi-socket boxes).  *out_node = the node, -1 if unknown. */
smgx_status smgx_bind_numa(int device_id, int* out_node, char** err);
void* smgx_alloc_pinned(size_t bytes);                                  /* page-locked host memory for hot-path buffers */
void smgx_free_pinned(void* ptr);

/* ---- fleet: the `&[Arc<dyn Worker>]` slice select_worker receives ----------------------------------------- */
/* Defines the worker slice for `model_key` (normalize_model_key: "" → "unknown", mod.rs:151-157) in slice order and
 * performs init_workers (cache_aware.rs:219-249).  Calling it again replaces the slice (trees are kept). */
smgx_status smgx_set_workers(smgx_policy* p, const char* model_key, const char* const* urls, uint32_t n, char** err);
/* Worker scalars read by the path (worker/worker.rs:151-153,187,208): load(), is_healthy(), circuit_breaker_can_execute().
 * `circuit_ok` may be NULL (= all 1).  The snapshot applies to every later select call until replaced. */
smgx_status smgx_set_fleet_state(smgx_policy* p, const char* model_key, const uint64_t* loads, const uint8_t* healthy,
                                 const uint8_t* circuit_ok, uint32_t n, char** err);
/* add_worker_by_url / remove_worker_by_url (cache_aware.rs:269-308; removal is a no-op in the reference too). */
smgx_status smgx_add_worker(smgx_policy* p, const char* model_key, const char* url, char** err);
smgx_status smgx_remove_worker(smgx_policy* p, const char* model_key, const char* url, char** err);
/* increment_processed() counters accumulated per slice index since the last call; out may be NULL to reset. */
smgx_status smgx_take_processed(smgx_policy* p, const char* model_key, uint64_t* out_counts, uint32_t n, char** err);

/* ---- event-driven index: kv_index::PositionalIndexer (crates/kv_index/src/event_tree.rs) ------------------- */
/* set_kv_event_monitor(Some/None) (cache_aware.rs:213-215). */
smgx_status smgx_set_kv_event_monitor(smgx_policy* p, int present, char** err);
/* KvEventMonitor creates one indexer per model (kv_event_monitor.rs); jump_size default there is 64 (:31). */
smgx_status smgx_indexer_create(smgx_policy* p, const char* model_key, uint32_t jump_size, char** err);
smgx_status smgx_indexer_set_block_size(smgx_policy* p, const char* model_key, uint32_t block_size, char** err); /* learned block size */
smgx_status smgx_indexer_intern_worker(smgx_policy* p, const char* model_key, const char* url, uint32_t* out_id, char** err);      /* :509-525 */
smgx_status smgx_indexer_worker_id(smgx_policy* p, const char* model_key, const char* url, int64_t* out_id /* -1 = None */, char** err); /* :294 */
/* apply_stored (:305-366).  StoredBlock = {seq_hash, content_hash}; parent_seq_hash NULL = None.
 * Returns SMGX_WORKER_NOT_TRACKED / SMGX_PARENT_BLOCK_NOT_FOUND so the caller can replicate the fresh-chain
 * fallback of kv_event_monitor.rs:559-571.  The per-worker WorkerBlockMap (:246) lives inside the policy. */
smgx_status smgx_indexer_apply_stored(smgx_policy* p, const char* model_key, uint32_t worker_id, const uint64_t* seq_hashes,
                                      const uint64_t* content_hashes, uint32_t n_blocks, const uint64_t* parent_seq_hash, char** err);
/* Same, hashing `token_ids` (n_blocks × block_size u32) like convert_kv_block (kv_event_monitor.rs:592-597). */
smgx_status smgx_indexer_apply_stored_tokens(smgx_policy* p, const char* model_key, uint32_t worker_id, const uint64_t* seq_hashes,
                                             const uint32_t* token_ids, uint32_t block_size, uint32_t n_blocks,
                                             const uint64_t* parent_seq_hash, char** err);
smgx_status smgx_indexer_apply_removed(smgx_policy* p, const char* model_key, uint32_t worker_id, const uint64_t* seq_hashes, uint32_t n, char** err); /* :380-404 */
smgx_status smgx_indexer_apply_cleared(smgx_policy* p, const char* model_key, uint32_t worker_id, char** err);  /* :410-420 */
smgx_status smgx_indexer_remove_worker(smgx_policy* p, const char* model_key, uint32_t worker_id, char** err);  /* :426-435 */
smgx_status smgx_indexer_current_size(smgx_policy* p, const char* model_key, uint64_t* out, char** err);        /* :438-444 */
smgx_status smgx_indexer_entry_count(smgx_policy* p, const char* model_key, uint64_t* out, char** err);         /* index.len() */
/* KvEventMonitor::apply_event for a batch (worker/kv_event_monitor.rs:525-597; proto crates/grpc_client/proto/common.proto:41-58).
 * Event e of kind STORED carries blocks [first_block, first_block + n_blocks) of the flat block arrays: block j has the engine's
 * block_hash[j] (i64, reinterpreted as u64 like SequenceHash::from) and token_ids[block_tok_offsets[j] .. block_tok_offsets[j+1]);
 * REMOVED uses block_hash[...] only; CLEARED nothing.  Content hashes of all stored blocks are computed in one GPU launch; events are
 * applied in order; a Stored event whose parent is unknown is retried as a fresh chain, as the reference does (*out_fallbacks counts). */
typedef enum smgx_kv_event_kind { SMGX_KV_STORED = 0, SMGX_KV_REMOVED = 1, SMGX_KV_CLEARED = 2 } smgx_kv_event_kind;
typedef struct smgx_kv_event {
    uint32_t kind;               /* smgx_kv_event_kind */
    uint32_t worker_id;          /* from smgx_indexer_intern_worker */
    uint32_t first_block, n_blocks;
    int64_t parent_block_hash;   /* KvBlocksStored.parent_block_hash */
    uint32_t has_parent;
    uint32_t reserved;
} smgx_kv_event;
smgx_status smgx_kv_events_apply(smgx_policy* p, const char* model_key, const smgx_kv_event* events, uint32_t n_events, const int64_t* block_hashes,
                                 const uint32_t* block_tok_offsets, const uint32_t* token_ids, uint32_t n_blocks, uint32_t* out_fallbacks, char** err);

/* find_matches (:461) on the GPU: `content_hashes` (host) → per-worker overlap.  out_scores[w] = 0 means "absent from
 * OverlapScores.scores"; out_tree_sizes[w] is valid where out_scores[w] > 0.  Arrays hold `cap` entries (≥ worker count). */
smgx_status smgx_indexer_find_matches(smgx_policy* p, const char* model_key, const uint64_t* content_hashes, uint32_t n,
                                      int early_exit, uint32_t* out_scores, uint64_t* out_tree_sizes, uint32_t cap,
                                      uint32_t* out_n_workers, char** err);
/* compute_request_content_hashes (:141-151) on the GPU, for callers/tests that want the hashes themselves. */
smgx_status smgx_content_hashes(smgx_policy* p, const uint32_t* tokens, uint32_t n_tokens, uint32_t block_size,
                                uint64_t* out_hashes, uint32_t cap, uint32_t* out_n, char** err);

/* ---- approximate token tree: kv_index::TokenTree (crates/kv_index/src/token_tree.rs) ----------------------------- */
/* TokenTree::with_policy (:359): 0 LRU, 1 LFU, 2 FIFO, 3 MRU, 4 FILO, 5 Priority.  smgx_set_workers creates an LRU tree
 * per model (init_workers, cache_aware.rs:231-247); call this to (re)create it with another eviction policy. */
smgx_status smgx_tree_create(smgx_policy* p, const char* model_key, int eviction_policy, char** err);
smgx_status smgx_tree_insert_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, uint32_t n, const char* tenant, char** err); /* :401 */
/* match_prefix_with_counts (:615) on the GPU, incl. its touch side effects; out_tenant receives the tenant URL ("empty" when
 * nothing matched). */
smgx_status smgx_tree_match_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, uint32_t n, uint32_t* out_matched,
                                   uint32_t* out_input, char* out_tenant, uint32_t tenant_cap, char** err);
/* n inserts in one call (tree build / replay): sequence i = tokens[offsets[i] .. offsets[i+1]) for tenants[i]. */
smgx_status smgx_tree_insert_tokens_batch(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint64_t* offsets, uint32_t n,
                                          const char* const* tenants, char** err);
/* Read-only walk + pick (match_prefix_with_counts without its touches, then the select_worker_with_tokens decision) of
 * device-resident batches against the current tree; batch j runs on lane j % smgx_pipeline_depth().  The walk kernel on
 * its own — bench and capacity planning; routing goes through the select calls, which also apply the side effects. */
smgx_status smgx_tree_walk_many_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint32_t* const* d_tokens,
                                       const uint32_t* const* d_offsets, const uint32_t* n, int32_t* const* d_out_worker_idx,
                                       smgx_decision_info* const* d_out_info, char** err);
smgx_status smgx_tree_evict_tenant(smgx_policy* p, const char* model_key, const char* tenant, uint64_t max_tokens, char** err);  /* :798 */
smgx_status smgx_evict_cache(smgx_policy* p, uint64_t max_size, char** err);          /* CacheAwarePolicy::evict_cache (cache_aware.rs:311) */
smgx_status smgx_tree_tenant_size(smgx_policy* p, const char* model_key, const char* tenant, uint64_t* out, char** err);           /* :988 */
smgx_status smgx_tree_clear(smgx_policy* p, const char* model_key, char** err);                                                     /* :997 */
/* iter_entries (:1039) as text, one line per entry "tok,tok,…|tenant=ts;tenant=ts"; *out_text is callee-allocated (smgx_free_string). */
smgx_status smgx_tree_entries(smgx_policy* p, const char* model_key, char** out_text, char** err);
smgx_status smgx_set_tree_batch_mode(smgx_policy* p, uint32_t mode, char** err);

/* ---- string tree: kv_index::Tree (crates/kv_index/src/string_tree.rs), HTTP text routing ----------------------- */
/* Text is UTF-8 (Rust &str); counts are Unicode scalar values.  Mutations run on the host-authoritative tree inside the
 * library; smgx_stree_match walks the GPU mirror.  One tree per model key, created by smgx_set_workers / on first use. */
smgx_status smgx_stree_insert_text(smgx_policy* p, const char* model_key, const uint8_t* text, uint32_t n_bytes, const char* tenant, char** err); /* :393 */
/* match_prefix_with_counts (:561-649): matched / input char counts and the tenant ("empty" when the node has none). */
smgx_status smgx_stree_match(smgx_policy* p, const char* model_key, const uint8_t* text, uint32_t n_bytes, uint32_t* out_matched_chars,
                             uint32_t* out_input_chars, char* out_tenant, uint32_t tenant_cap, char** err);
/* prefix_match_tenant (:659-720) — not on the routing path; host walk.  Returns the matched prefix length in bytes. */
smgx_status smgx_stree_prefix_match_tenant(smgx_policy* p, const char* model_key, const uint8_t* text, uint32_t n_bytes, const char* tenant,
                                           uint32_t* out_matched_bytes, char** err);
/* "tenant=chars\n" lines: maintained != 0 → get_tenant_char_count (:855), else get_used_size_per_tenant (:862). smgx_free_string. */
smgx_status smgx_stree_sizes(smgx_policy* p, const char* model_key, int maintained, char** out_text, char** err);
/* iter_entries (:1116-1221), pre-order, children in char order: records "path \x1f tenant=epoch;... \x1e". smgx_free_string. */
smgx_status smgx_stree_entries(smgx_policy* p, const char* model_key, char** out_text, uint64_t* out_len, char** err);
/* Read-only walk + pick of device-resident text batches (the string-tree kernel on its own — bench); d_out_node[j][i] = node the walk ended on. */
smgx_status smgx_stree_walk_many_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint8_t* const* d_text,
                                        const uint32_t* const* d_offsets, const uint32_t* n, int32_t* const* d_out_worker_idx,
                                        smgx_decision_info* const* d_out_info, uint32_t* const* d_out_node, char** err);
/* Mesh wire format (SURVEY §8f rank 3): kv_index::snapshot::TreeSnapshot (crates/kv_index/src/snapshot.rs:18-52) in bincode 1.3 default
 * encoding — u64-LE node count, then per node in pre-order { u64 len + UTF-8 edge, u64 n + n × { u64 len + tenant, u64 epoch }, u32
 * child_count }, children in char order (tenants in name order, where DashMap order is arbitrary).
 *   smgx_stree_snapshot        Tree::snapshot().to_bytes()       (string_tree.rs:1066-1102; *out_bytes is freed with smgx_free_string)
 *   smgx_stree_load_snapshot   Tree::from_snapshot(from_bytes())  (:1228-1309): REPLACES the model's string tree
 *   smgx_stree_merge_snapshot  Tree::merge_snapshot               (:1318-1545): remote wins on a newer epoch; three edge cases
 * Malformed bytes → SMGX_INVALID_ARGUMENT, the tree is left untouched.  No epoch is drawn by any of the three. */
smgx_status smgx_stree_snapshot(smgx_policy* p, const char* model_key, char** out_bytes, uint64_t* out_len, char** err);
smgx_status smgx_stree_load_snapshot(smgx_policy* p, const char* model_key, const uint8_t* bytes, uint64_t n_bytes, char** err);
smgx_status smgx_stree_merge_snapshot(smgx_policy* p, const char* model_key, const uint8_t* bytes, uint64_t n_bytes, char** err);
smgx_status smgx_stree_clear(smgx_policy* p, const char* model_key, char** err);
smgx_status smgx_stree_node_count(smgx_policy* p, const char* model_key, uint64_t* out, char** err);

/* ---- mesh path hashes and the hash_index side effect (crates/mesh/src/hash.rs:22-52; cache_aware.rs:95-101) ------------- */
/* hash_token_path / hash_node_path for a batch on the GPU: BLAKE3 of the little-endian u32 ids (or the UTF-8 bytes) of request i,
 * low 8 digest bytes little-endian, 0 remapped to 1.  The tree-mode select calls compute these themselves and record
 * hash(full request) → matched prefix, exactly where the reference does (:397-401, :420-424, :881-886, :950-956);
 * smgx_evict_cache clears a model's map when it outgrows max_size (:335-351). */
smgx_status smgx_hash_token_paths(smgx_policy* p, const uint32_t* tokens, const uint32_t* offsets, uint32_t n, uint64_t* out_hashes, char** err);
smgx_status smgx_hash_node_paths(smgx_policy* p, const uint8_t* text, const uint32_t* offsets, uint32_t n, uint64_t* out_hashes, char** err);
/* text_kind 0: token_tree map (values are u32 ids), 1: string_tree map (values are UTF-8 bytes). */
/* ---- TreeHandle (cache_aware.rs:454-645): what the mesh adapter calls on the policy -------------------------------------------------
 *   apply_known_remote_insert (:499-551)  smgx_tree_apply_known_remote_insert: *out_known = 1 and the stored matched prefix gains
 *                                         `worker_url` as a tenant when hash_index[model] resolves `node_hash`; 0 otherwise (ask a peer for repair)
 *   open_repair_stream (:553-573)         smgx_stree_entries / smgx_tree_entries (iter_entries in the trees' deterministic pre-order)
 *   apply_repair_page (:575-645)          smgx_tree_apply_repair_page: entries whose kind differs from tree_kind are skipped; the tree is
 *                                         created if missing; every applied entry seeds hash_index with its blake3 path hash (GPU)
 * tree_kind / smgx_repair_entry.kind: 0 = TreeKind::String (UTF-8 bytes), 1 = TreeKind::Token (u32 ids). */
typedef struct smgx_repair_entry {
    uint32_t kind;                 /* 0 = RepairEntry::String, 1 = RepairEntry::Token */
    uint32_t len;                  /* bytes (String) or tokens (Token) */
    const void* data;
    const char* const* tenants;    /* the entry's tenant URLs (epochs are not used by apply_repair_page) */
    uint32_t n_tenants;
    uint32_t reserved;
} smgx_repair_entry;
smgx_status smgx_tree_apply_known_remote_insert(smgx_policy* p, const char* model_key, int tree_kind, uint64_t node_hash, const char* worker_url,
                                                int* out_known, char** err);
smgx_status smgx_tree_apply_repair_page(smgx_policy* p, const char* model_key, int tree_kind, const smgx_repair_entry* entries, uint32_t n,
                                        uint32_t* out_applied, char** err);
smgx_status smgx_hash_index_size(smgx_policy* p, const char* model_key, int text_kind, uint64_t* out, char** err);
smgx_status smgx_hash_index_get(smgx_policy* p, const char* model_key, int text_kind, uint64_t path_hash, void* out, uint32_t cap_bytes,
                                uint32_t* out_bytes, int* out_found, char** err);

/* ---- adjacent policy on the same plumbing: power_of_two (model_gateway/src/policies/power_of_two.rs; SURVEY.md §8f rank 4) ----
 * PowerOfTwoPolicy::update_loads (:129-135): extends the cached url → load-response map; only effective_token_usage() (protocols worker.rs:1039-1044,
 * the mean token_usage over the DP ranks, 0.0 for an empty list) is read by select_worker, so that is what crosses the boundary. */
smgx_status smgx_power_of_two_update_loads(smgx_policy* p, const char* const* urls, const double* token_usage, uint32_t n, char** err);
/* PowerOfTwoPolicy::select_worker (:36-120) for n requests against the worker slice and fleet snapshot of `model_key` (smgx_set_workers +
 * smgx_set_fleet_state): None (-1) without a healthy worker, the only healthy worker if there is one, else two distinct candidates drawn
 * as idx1 = uniform(0..h), idx2 = (idx1 + 1 + uniform(0..h-1)) % h over the healthy indices, compared by token usage when BOTH have a cached
 * load response and by request count (Worker::load()) otherwise, first candidate on ties.  The reference draws from an unseedable
 * thread-local generator; here request i of the call uses draws 2i and 2i + 1 of the counter-based stream `seed` selects (csrc/power_of_two.cu),
 * so a caller advances `seed` per call.  out_pairs (2n, nullable): the two candidates, -1 -1 when none were drawn; out_metric (n, nullable):
 * 0 = request_count, 1 = token_usage, 2 = no comparison.  The router's own follow-ups stay on the host: increment_processed() (:110) on the pick. */
smgx_status smgx_power_of_two_select_batch(smgx_policy* p, const char* model_key, uint32_t n, uint64_t seed, int32_t* out_worker_idx, int32_t* out_pairs,
                                           uint8_t* out_metric, char** err);

/* ---- adjacent policy on the same plumbing: prefix_hash (model_gateway/src/policies/prefix_hash.rs; SURVEY.md §8f rank 4) ---- */
/* Which branch of PrefixHashPolicy::select_worker_impl produced the result (prefix_hash.rs:61-83), reported in
 * smgx_decision_info.branch by the smgx_prefix_hash_* calls (matched = 0, input = request length in tokens). */
typedef enum smgx_prefix_branch {
    SMGX_PH_NO_HEALTHY_WORKERS = 0,   /* empty slice or no is_healthy() worker → None (:143-145, :208-210) */
    SMGX_PH_NO_TOKENS = 1,            /* info.tokens None or empty → None               (:213-216)          */
    SMGX_PH_RING_HIT = 2,             /* ring worker passes load_ok                      (:169-171)          */
    SMGX_PH_LOAD_BALANCE_WALK = 3,    /* ring worker overloaded → least loaded acceptable worker, else itself (:173-187) */
    SMGX_PH_FALLBACK_LEAST_LOAD = 4   /* no ring / ring lookup failed → least loaded healthy (:192-199)      */
} smgx_prefix_branch;
/* PrefixHashConfig (prefix_hash.rs:38-58): defaults 256 tokens / 1.25. */
smgx_status smgx_prefix_hash_configure(smgx_policy* p, uint64_t prefix_token_count, double load_factor, char** err);
/* info.hash_ring for `model_key`: HashRing::new(urls) (worker/hash_ring.rs:45-70) — 150 virtual nodes per URL at
 * blake3("{url}#{vnode}")[..8] (hashed on the GPU), sorted by position (equal positions keep insertion order).  The ring is
 * independent of the worker slice, as in the reference (the registry rebuilds it when workers come and go); n = 0 gives the empty
 * ring, smgx_hash_ring_clear gives hash_ring = None. */
smgx_status smgx_hash_ring_set(smgx_policy* p, const char* model_key, const char* const* urls, uint32_t n, char** err);
smgx_status smgx_hash_ring_clear(smgx_policy* p, const char* model_key, char** err);
/* The sorted entries: out_pos[i], out_url[i] (index into the urls of smgx_hash_ring_set); *out_len = HashRing::len(). */
smgx_status smgx_hash_ring_entries(smgx_policy* p, const char* model_key, uint64_t* out_pos, uint32_t* out_url, uint32_t cap, uint32_t* out_len, char** err);
/* HashRing::find_healthy_url (hash_ring.rs:102-134) for n keys: key i = keys[key_offsets[i] .. key_offsets[i+1]) (any bytes),
 * url_ok[u] = is_healthy(url u of the ring).  out_url[i] = ring URL index or -1 (None). */
smgx_status smgx_hash_ring_find_healthy(smgx_policy* p, const char* model_key, const uint8_t* keys, const uint32_t* key_offsets, uint32_t n,
                                        const uint8_t* url_ok, int32_t* out_url, char** err);
/* compute_prefix_hash (prefix_hash.rs:106-113) of every request: xxh3_64 of the first min(len, prefix_token_count) token ids. */
smgx_status smgx_prefix_hashes(smgx_policy* p, const uint32_t* tokens, const uint32_t* offsets, uint32_t n, uint64_t* out_hashes, char** err);
/* PrefixHashPolicy::select_worker (prefix_hash.rs:225-229) for a batch against the worker slice and fleet snapshot of `model_key`
 * (smgx_set_workers / smgx_set_fleet_state; only is_healthy() and load() are read, :140, :148) and the model's ring.
 * has_tokens[i] = 0 means info.tokens = None for request i (NULL: every request carries tokens).  Host buffers; only the hashed
 * prefix of each request crosses PCIe. */
smgx_status smgx_prefix_hash_select_batch_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n,
                                                 const uint8_t* has_tokens, int32_t* out_worker_idx, smgx_decision_info* out_info, char** err);
/* Device-resident form, up to 32 batches per launch (batch k = d_tokens[k], d_offsets[k], n[k] → d_out_worker_idx[k]); asynchronous
 * on lane 0 — bracket with smgx_timer_* / smgx_synchronize. */
smgx_status smgx_prefix_hash_select_many_tokens_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint32_t* const* d_tokens,
                                                       const uint32_t* const* d_offsets, const uint32_t* n, int32_t* const* d_out_worker_idx, char** err);

/* ---- adjacent policy on the same plumbing: consistent_hashing (model_gateway/src/policies/consistent_hashing.rs) ---- */
/* Which branch of ConsistentHashingPolicy::select_worker_impl produced the result, in Branch::as_str order (:31-51). */
typedef enum smgx_ch_branch {
    SMGX_CH_NO_HEALTHY_WORKERS = 0,   /* empty slice, no healthy worker for the key, or no healthy worker for the random pick */
    SMGX_CH_TARGET_WORKER_HIT = 1,    /* X-SMG-Target-Worker names a healthy slice index (:128-137)                           */
    SMGX_CH_TARGET_WORKER_MISS = 2,   /* X-SMG-Target-Worker is not a usize, out of range or unhealthy → None                 */
    SMGX_CH_ROUTING_KEY_HIT = 3,      /* X-SMG-Routing-Key, else the implicit authorization / x-forwarded-for / cookie key     */
    SMGX_CH_RANDOM_FALLBACK = 4       /* no key: a uniformly drawn is_healthy() worker (:163-185)                              */
} smgx_ch_branch;
/* ConsistentHashingPolicy::select_worker_impl (:116-186) for n requests against the worker slice and fleet snapshot of `model_key`
 * (smgx_set_workers + smgx_set_fleet_state; only is_healthy() is read, the circuit breaker is not) and the model's ring: the ring of
 * smgx_hash_ring_set, none before it or after smgx_hash_ring_clear (info.hash_ring = None → the modulo fallback over the sorted healthy
 * indices, one per URL).  Headers of request i: header h = values[offsets[5i+h] .. offsets[5i+h+1]) for h = 0 x-smg-target-worker,
 * 1 x-smg-routing-key, 2 authorization, 3 x-forwarded-for, 4 cookie; present[i] bit h = HeaderMap::get(name h) returned Some (the first
 * value of a repeated header; info.headers = None ⇔ 0).  A value is used only if every byte is \t or 0x20..=0x7E (HeaderValue::to_str)
 * and it is non-empty; the target worker is parsed as usize::from_str.  The implicit key is the first PRESENT of authorization,
 * x-forwarded-for, cookie, and an empty or non-visible value there goes to the random fallback.  The reference draws the random fallback
 * from an unseedable thread-local generator; here request i uses draw i of the counter-based stream `seed` selects (the power_of_two
 * stream), mapped to ⌊x·h / 2^64⌋ over the h healthy workers in slice order, so a caller advances `seed` per call.
 * Host buffers; offsets (5n + 1, non-decreasing) need not start at 0 and only values[offsets[0] .. offsets[5n]) crosses PCIe.  Any present
 * x-smg-routing-key, authorization, x-forwarded-for or cookie value longer than 2 MiB is SMGX_INVALID_ARGUMENT for the whole call, whether
 * or not it would be the key used (the check runs on the offsets, before any byte is read); the target-worker value has no limit.  out_branch (n, nullable): smgx_ch_branch; out_key_pos (n, nullable): blake3(key)[..8] LE of
 * the key used, 0 when no key was hashed.  No pick reads a load, so load feedback (smgx_set_load_feedback_policies) does not apply. */
smgx_status smgx_consistent_hashing_select_batch(smgx_policy* p, const char* model_key, uint32_t n, const uint8_t* values, const uint32_t* offsets,
                                                 const uint8_t* present, uint64_t seed, int32_t* out_worker_idx, uint8_t* out_branch,
                                                 uint64_t* out_key_pos, char** err);

/* ---- HTTP text routing: select_worker with info.request_text = Some(text), info.tokens = None ------------------ */
/* select_worker_with_text (cache_aware.rs:907-974) and the imbalanced path's string-tree update (:403-425) for a batch:
 * request i = text[offsets[i] .. offsets[i+1]) (valid UTF-8).  match_rate = matched chars / input chars (f32, strict >).
 * out_info[i].matched / .input are char counts.  Batch serialisation: smgx_tree_batch_mode. */
smgx_status smgx_select_batch_request_text(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                           int32_t* out_worker_idx, smgx_decision_info* out_info, char** err);

/* ---- tokenizer: Tokenizer::encode for tiktoken-style models (crates/tokenizer/src/tiktoken.rs) ----------------- */
/* The pre-tokenizer regex a tokenizer splits ordinary text with:
 *   SMGX_PRETOK_CL100K  CL100K_BASE_PATTERN (tiktoken.rs:28): cl100k_base, and the Llama-3 Split regex of tokenizer.json files;
 *   SMGX_PRETOK_R50K    tiktoken's GPT-2 pattern r50k_pat_str: r50k_base, p50k_base, p50k_edit, and tokenizer.json files whose
 *                       pre-tokenizer is ByteLevel(use_regex = true, add_prefix_space = false) alone;
 *   SMGX_PRETOK_QWEN2   the Qwen2 Split regex: the cl100k pattern with \p{N} in place of \p{N}{1,3} (every digit is a piece);
 *   SMGX_PRETOK_DEEPSEEK  the chain of three Isolated Splits of DeepSeek V2 / V2.5 / Coder-V2 / V3 / V3.1 / R1 tokenizer.json files:
 *                       \p{N}{1,3}, then kana/CJK runs [一-龥぀-ゟ゠-ヿ]+, then the DeepSeek word regex on every piece (bpe.cuh).
 * Any other value (3 included) is SMGX_INVALID_ARGUMENT. */
typedef enum smgx_pretokenizer {
    SMGX_PRETOK_CL100K = 0, SMGX_PRETOK_R50K = 1, SMGX_PRETOK_QWEN2 = 2, SMGX_PRETOK_DEEPSEEK = 4
} smgx_pretokenizer;
/* The tokenizer.json normalizer applied to the text between special tokens before it is split:
 *   SMGX_NORMALIZER_NONE  none;
 *   SMGX_NORMALIZER_NFC   {"type": "NFC"} (Qwen2 and later), with the Unicode tables of the `tokenizers` crate.
 * Special-token strings are matched on the raw text (added tokens with normalized = false).  Any other value is
 * SMGX_INVALID_ARGUMENT. */
typedef enum smgx_normalizer { SMGX_NORMALIZER_NONE = 0, SMGX_NORMALIZER_NFC = 1 } smgx_normalizer;
/* TiktokenTokenizer::from_file (tiktoken.rs:219-268): `path` holds lines of `base64(token) rank` (load_tiktoken_bpe, :346-367);
 * `special_strs/special_ids` = the added_tokens_decoder entries that become CoreBPE's special-token encoder (:234-238).
 * The pre-tokenizer is CL100K_BASE_PATTERN (:28); the _ex form takes it as an argument.  One tokenizer per model key, so one
 * policy can hold models with different pre-tokenizers. */
smgx_status smgx_tokenizer_load_tiktoken_file(smgx_policy* p, const char* model_key, const char* path, const char* const* special_strs,
                                              const uint32_t* special_ids, uint32_t n_special, char** err);
smgx_status smgx_tokenizer_load_tiktoken_file_ex(smgx_policy* p, const char* model_key, const char* path, const char* const* special_strs,
                                                 const uint32_t* special_ids, uint32_t n_special, smgx_pretokenizer pretokenizer, char** err);
/* Same from memory: token i = blob[tok_offsets[i] .. tok_offsets[i+1]) with rank ranks[i]. */
smgx_status smgx_tokenizer_load_tiktoken(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets,
                                         const uint32_t* ranks, uint32_t n_tokens, const char* const* special_strs,
                                         const uint32_t* special_ids, uint32_t n_special, char** err);
smgx_status smgx_tokenizer_load_tiktoken_ex(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets,
                                            const uint32_t* ranks, uint32_t n_tokens, const char* const* special_strs,
                                            const uint32_t* special_ids, uint32_t n_special, smgx_pretokenizer pretokenizer, char** err);
/* HuggingFaceTokenizer (crates/tokenizer/src/huggingface.rs:310-316 → crate `tokenizers`), byte-level BPE family whose tokenizer.json
 * has: no normalizer; pre_tokenizer = Split(Regex = the cl100k pattern above, Isolated) + ByteLevel(use_regex = false) — Llama 3 and
 * kin — or, with SMGX_PRETOK_R50K through the _ex form, ByteLevel(use_regex = true, add_prefix_space = false) alone — GPT-2 and kin,
 * or, with SMGX_PRETOK_DEEPSEEK, DeepSeek's Sequence of three Splits + ByteLevel(use_regex = false) (its empty-Sequence normalizer is
 * the identity: load it with SMGX_NORMALIZER_NONE);
 * model.type = "BPE" without dropout / unk / byte_fallback.  The caller parses the JSON (serde_json in the gateway,
 * smg_b200/policy.py here) and hands over: token i = blob[tok_offsets[i] .. tok_offsets[i+1]) as RAW bytes (byte-level chars mapped
 * back) with id ids[i]; `merges` = n_merges (left id, right id) pairs in priority order; model.ignore_merges; added_tokens as specials. */
smgx_status smgx_tokenizer_load_bpe_merges(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                           uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, int ignore_merges,
                                           const char* const* special_strs, const uint32_t* special_ids, uint32_t n_special, char** err);
smgx_status smgx_tokenizer_load_bpe_merges_ex(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                              uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, int ignore_merges,
                                              const char* const* special_strs, const uint32_t* special_ids, uint32_t n_special,
                                              smgx_pretokenizer pretokenizer, char** err);
/* The same with a normalizer (tokenizer.json `normalizer`); the _ex form forwards with SMGX_NORMALIZER_NONE. */
smgx_status smgx_tokenizer_load_bpe_merges_norm(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                                uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, int ignore_merges,
                                                const char* const* special_strs, const uint32_t* special_ids, uint32_t n_special,
                                                smgx_pretokenizer pretokenizer, smgx_normalizer normalizer, char** err);
/* SentencePiece-style BPE tokenizer.json files (Llama 2, CodeLlama, Mistral, Mixtral, TinyLlama): model.type = "BPE" with
 * byte_fallback = true, the 256 tokens "<0x00>" … "<0xFF>" and "▁" (U+2581) in the vocabulary, no dropout / continuing_subword_prefix /
 * end_of_word_suffix, ignore_merges = false.  Spaces become ▁ and a stretch of text between added tokens starts with ▁, in one of two shapes:
 *   SMGX_SP_LEGACY     normalizer Sequence[Prepend("▁"), Replace(" " → "▁")], pre_tokenizer null: every non-empty stretch gets a ▁ in
 *                      front; prepend_scheme must be SMGX_PREPEND_ALWAYS and split 0;
 *   SMGX_SP_METASPACE  normalizer null, pre_tokenizer Metaspace(replacement "▁", prepend_scheme, split): a ▁ is prepended unless the
 *                      stretch already starts with one — SMGX_PREPEND_FIRST only to the stretch at offset 0 of the text, SMGX_PREPEND_NEVER
 *                      never; split = 1 cuts the stretch before every ▁.
 * Tokens are RAW UTF-8 strings (no byte-level mapping), merges and specials as for smgx_tokenizer_load_bpe_merges_ex; added tokens are
 * matched on the raw text.  Initial symbols are code points; one that is not in the vocabulary becomes the <0xXX> tokens of its bytes.
 * Without split, the GPU merges the pieces of a stretch cut before every ▁ that follows another character; the load refuses
 * (SMGX_TOKENIZATION_ERROR, naming the merge) a vocabulary with a merge (a, b) where `a` does not end in ▁ and `b` starts with ▁, the one
 * case where that cut would change the result.  A missing ▁ or byte token is SMGX_TOKENIZATION_ERROR; an unknown enum value, split other
 * than 0 / 1 or a null pointer is SMGX_INVALID_ARGUMENT. */
typedef enum smgx_sp_shape { SMGX_SP_LEGACY = 0, SMGX_SP_METASPACE = 1 } smgx_sp_shape;
typedef enum smgx_prepend_scheme { SMGX_PREPEND_NEVER = 0, SMGX_PREPEND_FIRST = 1, SMGX_PREPEND_ALWAYS = 2 } smgx_prepend_scheme;
smgx_status smgx_tokenizer_load_bpe_metaspace(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                              uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, const char* const* special_strs,
                                              const uint32_t* special_ids, uint32_t n_special, smgx_sp_shape shape, smgx_prepend_scheme prepend_scheme,
                                              int split, char** err);
/* Encoder::encode_batch (tiktoken.rs:464-469) on the GPU: text i = text[offsets[i] .. offsets[i+1]) (UTF-8, already
 * chat-template-rendered; special-token strings are recognised, tiktoken.rs:446-460).  Writes the ragged token ids and
 * out_tok_offsets[n+1]; `cap_tokens` = capacity of out_tokens: total text bytes is always enough for a tokenizer without a
 * normalizer, 3 × total text bytes for a normalizing one (NFC can grow text threefold, e.g. U+1D160 → three code points), and
 * 2 × total text bytes for a SentencePiece-style one (a stretch of L bytes has at most L + 1 initial symbols: the prepended ▁). */
smgx_status smgx_tokenize_batch(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                uint32_t* out_tokens, uint32_t* out_tok_offsets, uint32_t cap_tokens, char** err);
/* The whole hot path in one call: tokenize on the device → cache-aware pick; the token ids never visit the host unless
 * out_tokens / out_tok_offsets are given (the gateway forwards them to the engine). */
smgx_status smgx_select_batch_text(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                   int32_t* out_worker_idx, smgx_decision_info* out_info, uint32_t* out_tokens,
                                   uint32_t* out_tok_offsets, uint32_t cap_tokens, char** err);

/* ---- the hot call: LoadBalancingPolicy::select_worker, batched (cache_aware.rs:648-690) -------------------- */
/* n requests, request i = tokens[offsets[i] .. offsets[i+1]) (SelectWorkerInfo.tokens = Some).  All requests see the
 * fleet snapshot and index state current at submission.  out_worker_idx[i] = index into the slice given to
 * smgx_set_workers, or -1 for None.  `out_info` may be NULL.  Host buffers; the call copies H2D, runs the kernels and
 * copies the result back before returning. */
smgx_status smgx_select_batch_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets,
                                     uint32_t n, int32_t* out_worker_idx, smgx_decision_info* out_info, char** err);
/* Batch semantics of the event-driven mode with respect to load():
 *   off (default): every request of a batch is decided against ONE fleet snapshot (the state at submission).
 *   on: "request i sees the snapshot plus the picks of requests < i" — after each pick the chosen worker's load is bumped before the next
 *       request of the call is decided, which is what the reference's request stream does (one select_worker per request, then
 *       WorkerLoadGuard::new → increment_load, routers/http/router.rs:319-321, worker/worker.rs:1067-1070): min-load picks spread over the
 *       fleet instead of all landing on one worker, (score, load) tie-breaks read the running loads and the f32 imbalance gate is
 *       re-evaluated per request.  Batches handed over in one smgx_select_many_tokens_device call form one stream.  The bumps are not
 *       kept: the next call starts from the snapshot of its own smgx_set_fleet_state.  Not available with duplicate URLs in the slice,
 *       for mapped submissions or for sharded candidates.
 * smgx_set_load_feedback and smgx_set_load_feedback_policies set ONE state and the last call wins: smgx_set_load_feedback(p, e) is
 * the mask "event-driven calls only, if e", smgx_set_load_feedback_policies(p, 0) turns every stream off. */
smgx_status smgx_set_load_feedback(smgx_policy* p, int enabled, char** err);
/* Load feedback per policy: the gateway names the picks its router follows with a WorkerLoadGuard — the HTTP router guards cache_aware
 * picks (routers/http/router.rs:319-321), the gRPC router every pick (routers/grpc/context.rs:248-259).
 *   SMGX_FEEDBACK_CACHE_AWARE: every cache_aware mode — the event-driven calls as smgx_set_load_feedback(p, 1) does, and the token-tree and
 *       string-tree modes (smgx_select_batch_tokens, smgx_submit_tokens, smgx_select_batch_text, smgx_submit_text,
 *       smgx_select_batch_request_text, an event-mode model whose indexer is empty).  Request i of a call is decided as select_worker would
 *       decide it with the snapshot loads plus one per pick of requests < i: the f32 imbalance gate, the min-load picks and the fallback to
 *       the first healthy worker read the running loads.  Not with SMGX_TREE_BATCH_SNAPSHOT (no interleaving of concurrent select_worker
 *       calls reads snapshot trees with streamed loads): the setter, and a tree-mode call that meets the combination, return
 *       SMGX_INVALID_ARGUMENT.
 *   SMGX_FEEDBACK_PREFIX_HASH: smgx_prefix_hash_select_batch_tokens and smgx_prefix_hash_select_many_tokens_device (every batch of one call
 *       forms one stream): the bound (Σ load + 1) / n × load_factor, the ring worker's load_ok and the least loaded fallback read the running loads.
 *   SMGX_FEEDBACK_POWER_OF_TWO: smgx_power_of_two_select_batch: same draws and pairs; the request-count comparison reads the running loads.
 * The gRPC router sets all three bits, the HTTP router SMGX_FEEDBACK_CACHE_AWARE only.  The prefix_hash and power_of_two passes keep the
 * running loads in shared memory: a worker slice of more than 25 600 entries is SMGX_INVALID_ARGUMENT with their bit set.
 * The bumps are not kept after the call.  Any other bit is SMGX_INVALID_ARGUMENT. */
#define SMGX_FEEDBACK_CACHE_AWARE 1u
#define SMGX_FEEDBACK_PREFIX_HASH 2u
#define SMGX_FEEDBACK_POWER_OF_TWO 4u
smgx_status smgx_set_load_feedback_policies(smgx_policy* p, uint32_t mask, char** err);
/* Pipelined form for the host batcher: up to smgx_pipeline_depth() submissions may be in flight; each owns a stream
 * and device staging.  Buffers must stay valid (and should be pinned) until smgx_wait(ticket) returns.
 * Each submission is decided against the index, fleet snapshot, worker slice and routing mode current when it is submitted; index and
 * fleet changes made while it is in flight do not reach it, and tickets may be waited for in any order.  With every lane in flight a
 * submission returns SMGX_BUSY before it changes anything (no tree insert, nothing counted).  A submission of n = 0 requests still
 * returns a ticket.  Waiting for an unknown ticket, or a second time for the same ticket, is SMGX_INVALID_ARGUMENT.
 * increment_processed(): the picks of an event-mode submission are credited when smgx_wait returns for its ticket (smgx_take_processed
 * in between does not count them yet), and not at all if smgx_set_workers replaced the slice in between (it resets the counters);
 * tree-mode submissions complete inside the call and are credited there.
 * Load feedback with a token tree: the tree update that select_worker_min_load owes for the picks of a submission that took the
 * imbalanced branch is applied when its ticket is waited for, so the tree receives those requests in wait order. */
uint32_t smgx_pipeline_depth(const smgx_policy* p);
smgx_status smgx_submit_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n,
                               int32_t* out_worker_idx, smgx_decision_info* out_info, uint64_t* out_ticket, char** err);
smgx_status smgx_wait(smgx_policy* p, uint64_t ticket, char** err);

/* Latency path (small batches, per-request callers): zero-copy.  `tokens`, `offsets`, `out_worker_idx`, `out_info` and `done_flag` must
 * live in memory from smgx_alloc_pinned (device-visible at the same address).  The kernel reads the requests in place over PCIe, stores
 * the picks straight into out_worker_idx and finally stores `done_value` to *done_flag (release, system scope): the caller spins on the
 * flag — no staging copy, no stream synchronisation, no ticket, no lane is held.  Requests longer than max_request_tokens (0 = the
 * policy's max_tokens_per_request) get pick -1 / branch 255.  Event-driven mode only: SMGX_NOT_FOUND when the model is currently routed
 * through a tree (those modes mutate host state; use smgx_submit_tokens).  increment_processed() accounting is left to the caller. */
smgx_status smgx_submit_tokens_mapped(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n,
                                      uint32_t max_request_tokens, int32_t* out_worker_idx, smgx_decision_info* out_info, uint64_t* done_flag,
                                      uint64_t done_value, char** err);

/* Same for rendered text (smgx_select_batch_text without the token read-back): H2D, GPU tokenize, pick and D2H ride one lane. */
smgx_status smgx_submit_text(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                             int32_t* out_worker_idx, smgx_decision_info* out_info, uint64_t* out_ticket, char** err);

/* Device-resident form (inputs already in HBM; used by bench.py's kernel-only leg and by callers that tokenize on
 * the GPU).  Pointers are device pointers on the policy's device; asynchronous on the policy's stream `lane`
 * (0 ≤ lane < smgx_pipeline_depth()).  `max_request_tokens` bounds the longest request of the batch (sizes the per-warp
 * shared-memory scratch; 0 = config max_tokens_per_request; a longer request is reported by smgx_synchronize).
 * d_out_info may be NULL. */
smgx_status smgx_select_batch_tokens_device(smgx_policy* p, const char* model_key, uint32_t lane, const uint32_t* d_tokens,
                                            const uint32_t* d_offsets, uint32_t n, uint32_t max_request_tokens,
                                            int32_t* d_out_worker_idx, smgx_decision_info* d_out_info, char** err);
/* Several ready device-resident batches at once (what the host batcher hands over when more than one batch is queued):
 * batch j is enqueued on lane j % smgx_pipeline_depth(), so consecutive batches overlap on the GPU. */
smgx_status smgx_select_many_tokens_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint32_t* const* d_tokens,
                                           const uint32_t* const* d_offsets, const uint32_t* n, uint32_t max_request_tokens,
                                           int32_t* const* d_out_worker_idx, char** err);
/* Sharded event-driven pick, step 1 (every rank, on its shard): per-request best local candidate + the shard's fleet summary.
 * All pointers are device pointers. */
smgx_status smgx_shard_candidates_device(smgx_policy* p, const char* model_key, uint32_t lane, const uint32_t* d_tokens,
                                         const uint32_t* d_offsets, uint32_t n, uint32_t max_request_tokens,
                                         smgx_shard_candidate* d_out_cand, smgx_shard_fleet* d_out_fleet, char** err);
/* Step 2 (every rank, after the exchange): d_cands = [world][n], d_fleets = [world], global_base[g] = global slice index of
 * shard g's first worker (host array).  Writes global slice indices (−1 = None). */
smgx_status smgx_shard_reduce_device(smgx_policy* p, uint32_t lane, const smgx_shard_candidate* d_cands, const smgx_shard_fleet* d_fleets,
                                     const uint32_t* global_base, uint32_t world, uint32_t n, int32_t* d_out_worker_idx,
                                     smgx_decision_info* d_out_info, char** err);

/* Peer-memory exchange (one process per GPU, NVLink): instead of handing the candidates to a collective, every rank creates one
 * symmetric gather buffer, the ranks swap CUDA IPC handles once (any host channel), and from then on one asynchronous call per
 * batch runs, in stream order and without host synchronisation: candidate kernels → stores into every rank's buffer + release
 * flag → wait for every rank's flag → merge.  All ranks must issue the same sequence of fused calls.  A peer that does not show up
 * within ≈20 s is reported by smgx_synchronize. */
#define SMGX_IPC_HANDLE_BYTES 64
smgx_status smgx_shard_exchange_create(smgx_policy* p, uint32_t world, uint32_t rank, uint32_t max_batch, uint8_t* out_handle /* 64 B */, char** err);
smgx_status smgx_shard_exchange_connect(smgx_policy* p, const uint8_t* handles /* world × 64 B, rank order */, char** err);
smgx_status smgx_shard_select_fused_device(smgx_policy* p, const char* model_key, uint32_t lane, const uint32_t* d_tokens, const uint32_t* d_offsets,
                                           uint32_t n, uint32_t max_request_tokens, const uint32_t* global_base /* host, world */,
                                           int32_t* d_out_worker_idx, smgx_decision_info* d_out_info, char** err);
void* smgx_device_alloc(smgx_policy* p, size_t bytes, char** err);
void smgx_device_free(smgx_policy* p, void* dptr);
smgx_status smgx_memcpy_h2d(smgx_policy* p, void* dptr, const void* host, size_t bytes, char** err);
smgx_status smgx_memcpy_d2h(smgx_policy* p, void* host, const void* dptr, size_t bytes, char** err);
smgx_status smgx_synchronize(smgx_policy* p, char** err);
/* CUDA-event timing on the launching stream (lane): start/stop bracket whatever is enqueued between them. */
smgx_status smgx_timer_start(smgx_policy* p, uint32_t lane, char** err);
smgx_status smgx_timer_stop_ms(smgx_policy* p, uint32_t lane, float* out_ms, char** err);
/* Same across ALL lanes: start is recorded on lane 0 and every other lane is made to wait for it; stop joins every lane
 * into lane 0 before recording the end event — so the interval covers work issued round-robin over the lanes. */
smgx_status smgx_timer_start_all(smgx_policy* p, char** err);
/* start_all behind a hold kernel of ~hold_us µs: work enqueued during the hold runs back to back afterwards, so the measured interval is GPU
 * execution only (no host launch latency between the start event and the first kernel). */
smgx_status smgx_timer_start_all_gated(smgx_policy* p, uint32_t hold_us, char** err);
smgx_status smgx_timer_start_gated(smgx_policy* p, uint32_t lane, uint32_t hold_us, char** err);
smgx_status smgx_stream_hold(smgx_policy* p, uint32_t lane, uint32_t hold_us, char** err);       /* only the hold kernel */   /* one lane; stop with smgx_timer_stop_ms(lane) */
smgx_status smgx_timer_stop_all_ms(smgx_policy* p, float* out_ms, char** err);
/* Process-wide switch between the implementations of the event-driven pick (A/B measurements, tests): path 0 (default) = hash kernel + search
 * kernel pair, the search launched as a programmatic dependent of the hash kernel; 1 = the warp-per-request family (simple / tiled / persistent
 * fused kernels); 2 = hash stream whose last CTA per 256-request group runs the search (event_hs_kernel); 3 = ONE launch of persistent CTAs, each
 * streaming its run of requests through a shared-memory ring (bulk async copies), hashing it and searching what it hashed (event_stream_kernel;
 * block size 16, ≤ 32 blocks per request, ≤ 64 interned workers — anything else runs the pair).  Mapped submissions and load-feedback batches always
 * run the persistent fused kernel.  min_blocks_per_sm: 0 = keep, 3 or 4 = occupancy variant of the fused kernel.
 * Environment: SMGX_EVENT_PATH=split|fused|hs|stream, SMGX_FUSED_MINB=3|4, SMGX_PDL=0 (no dependent launch), SMGX_SEARCH_RPC=128|160|192|256. */
void smgx_set_event_path(int path, int min_blocks_per_sm);
/* L2 prefetch flavour of the fused kernel: 0 none, 1 one bulk prefetch per request (default), 2 one prefetch per lane (SMGX_FUSED_PF). */
void smgx_set_fused_prefetch(int flavour);
/* Requests per warp of the tiled event kernel (8, 16 or 32; 0 = never use it) and the launch size from which it is used (requests; < 0 =
 * the default, tile × 4 × SM count).  Environment: SMGX_FUSED_TILE. */
void smgx_set_fused_tile(int tile, int64_t min_total);
/* The register event kernels (the default for plain picks on fleets of ≤ 64 workers at block size 16): one thread per request
 * (event_lane_kernel) for launches of at least 256 requests per SM, one warp per request (event_warp_kernel) below that, both with
 * event_slow_kernel for rare shapes.  0 = off, 4, 5 or 6 = on (the values once chose occupancy variants of the one-warp-per-request
 * kernel; they are accepted and all mean on).  Environment: SMGX_EVENT_SIMPLE. */
void smgx_set_event_simple(int min_blocks_per_sm);
/* Token stream of the tiled kernel: 0 = register double buffer, 4 / 8 = cp.async shared-memory ring of that many requests per warp
 * (SMGX_TILE_DEPTH). */
void smgx_set_tile_depth(int depth);
/* Number of smgx kernel launches issued by this policy so far (bench.py's gpu_launches). */
uint64_t smgx_kernel_launches(const smgx_policy* p);
/* Writes a buffer larger than L2 (bench hygiene between timed iterations). */
smgx_status smgx_flush_l2(smgx_policy* p, char** err);

#ifdef __cplusplus
}
#endif
#endif /* SMGX_H */
