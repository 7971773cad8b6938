// Kernel-facing structures and launch wrappers (implemented in event_kernels.cu).
#pragma once
#include <cstdint>

#include "common.h"
#include "event_index.h"

namespace smgx {

// Per-model fleet snapshot as the kernels see it.  Built on the device by fleet_prepare_kernel from the raw slice
// arrays the caller hands to smgx_set_fleet_state.  "id space" = PositionalIndexer worker ids; "slice space" =
// indices into the `&[Arc<dyn Worker>]` slice select_worker returns (cache_aware.rs:648).
struct FleetDerived {
    int32_t min_load_idx;    // first argmin load() over healthy (min_by_key → FIRST min); -1 when none healthy
    int32_t first_healthy;   // healthy_indices.first()
    uint32_t n_healthy;
    uint32_t imbalanced;     // (max-min) > abs_thr && (max as f32) > (min as f32 * rel_thr)   (cache_aware.rs:669-670)
    uint64_t min_load, max_load;   // over ALL workers; min_load = UINT64_MAX for an empty slice (worker-id shards)
    uint64_t min_healthy_load;   // load of min_load_idx (lets worker-id shards be merged, SURVEY §8e)
};
static_assert(sizeof(FleetDerived) == sizeof(smgx_shard_fleet), "smgx_shard_fleet mirrors FleetDerived");
struct FleetView {
    const FleetDerived* derived;
    const int32_t* slice_of_id;   // [id] → slice index or -1
    const uint64_t* load_of_id;   // [id] → load of that slice entry
    const uint64_t* elig;         // [words] bitset in id space: healthy && circuit_ok && present in the slice
};

struct FleetRaw {
    const uint64_t* loads;        // [n_slice]
    const uint8_t* flags;         // [n_slice] bit0 = is_healthy(), bit1 = circuit_breaker_can_execute()
    const int32_t* id_of_slice;   // [n_slice] → indexer worker id or -1
    uint32_t n_slice;
    uint32_t n_ids;               // interned workers
    uint32_t words;               // bitset words (id space)
    uint32_t has_dups;            // two slice entries share a URL (same indexer id): resolve in slice order, see fleet_prepare_kernel
    uint64_t abs_threshold;
    float rel_threshold;
};

void launch_fleet_prepare(const FleetRaw& raw, FleetDerived* d_derived, int32_t* d_slice_of_id, uint64_t* d_load_of_id,
                          uint64_t* d_elig, cudaStream_t stream);

// The event-driven pick for up to kMaxMultiBatches batches per launch (blockIdx.y = batch; descriptors travel in the
// kernel parameter block).  Two kernels in stream order:
// Default: event_fused_kernel — ONE persistent kernel, one warp per request, hash → jump search → argmax, the next request's
// tokens prefetched while the current one is probed.  SMGX_EVENT_PATH=split keeps the round-1 two-kernel form for A/B runs:
//   hash_blocks_kernel           K2b part 1: XXH3 content hash of every full block, one thread per block, streaming
//   event_search_{thread,warp}   K2b part 2 + K3: jump search over the positional index + argmax worker
//                                (one thread per request for fleets ≤ 64 interned workers, one warp per request above)
//   `hashes` is then a scratch of sum(n) × max_blocks u64 laid out [request][max_blocks], written and read back out of L2.
constexpr int kMaxMultiBatches = 32;
// MultiArgs.err_flag bit (OR-ed in): a request needed event_slow_kernel in a launch that skipped it (MultiArgs.skip_slow); its pick is not written
constexpr uint32_t kErrNoSlowKernel = 4;
// what the hash kernel leaves per request for the search kernel's first phase: the two hashes the jump search probes first and the
// request's length — one 32 B record instead of the chain offsets → hash row → slots
struct alignas(32) SearchRec { uint64_t h0, h1; uint32_t ntok, pad0; uint64_t pad1; };
struct BatchDesc {
    const uint32_t* tokens;        // device, ragged
    const uint32_t* offsets;       // device, n + 1
    int32_t* out_idx;              // device, n
    smgx_decision_info* out_info;  // device, n (nullable)
    uint32_t n;
    uint32_t hash_base;            // first row of this batch in the hash scratch
    smgx_shard_candidate* cand;    // non-null: worker-id-sharded fleet — emit this shard's best candidate instead of a pick
};
struct MultiArgs {
    BatchDesc b[kMaxMultiBatches];
    uint32_t count;
    uint32_t block_size;
    uint32_t max_blocks;           // row length of the hash scratch = max blocks per request
    uint64_t* hashes;              // split path only (nullptr on the fused path)
    uint32_t* err_flag;            // device: set to 1 when a request exceeds max_blocks
    // mapped (zero-copy) submissions: when done_flag != nullptr the last CTA to finish stores done_value there with system-scope release
    // semantics (the flag lives in pinned host memory the caller spins on); done_counter = device word counting finished CTAs (self-resetting)
    uint64_t* done_flag;
    uint64_t done_value;
    uint32_t* done_counter;
    // load-feedback mode (smgx_set_load_feedback): the fused kernel stores, per request, the eligible set of workers tied on the best
    // overlap score ([total][words] u64, id space) and that score instead of a pick; feedback_resolve_kernel then walks the requests in
    // order, each pick bumping its worker's load before the next request is decided (the router's WorkerLoadGuard, router.rs:319-321).
    // split path: the hash kernel warms L2 with the index slots the search kernel will probe first (positions 0 and min(jump, last))
    SearchRec* recs;               // [total] (split path)
    // concurrent split launch: the search kernel runs on a side stream AT THE SAME TIME as the hash kernel; its CTAs of batch y wait until the
    // hash CTAs of batch y have all counted themselves into ready[y] (cumulative counters, never reset: target = value to reach)
    uint32_t* ready;               // device [kMaxMultiBatches] (nullable: plain stream order)
    uint32_t ready_target[kMaxMultiBatches];
    const void* pf_slots;          // EventIndexView.slots (nullable)
    uint32_t pf_mask, pf_jump;
    uint32_t* slow_queue;          // event_lane_kernel / event_warp_kernel → event_slow_kernel: [0] = count, [1] = CTA exit counter (both zero between launches), [2 .. total + 1] = request indices (each request pushed at most once)
    // 1: no request of this launch can be queued for event_slow_kernel (the index view holds no Multi entry, max_blocks ≤ 32 and
    // max_blocks − 1 ≤ jump), so it is not launched; a request that still reaches the queue sets err_flag to kErrNoSlowKernel
    uint32_t skip_slow;
    uint64_t* fb_winsets;
    uint32_t* fb_scores;           // 0xFFFFFFFF = request longer than max_blocks
    // one-launch path (event_hs_kernel): per (batch, group of 256 requests) arrival counters, zero between launches
    uint32_t* group_count;         // device [kMaxMultiBatches][group_stride] (nullable: the pair runs)
    uint32_t dbg;                  // SMGX_STREAM_DBG (diagnostics of event_stream_kernel): 1 = release a stage only after hashing it, 2 = __threadfence before the search
    uint32_t group_stride;
    uint32_t total;                // sum of b[k].n  (b[k].hash_base = requests before batch k)
    uint32_t uniform_n;            // every batch has this many requests (0: look the batch up through hash_base)
};
// true: launch_event_select runs the one-kernel fused path (no hash scratch needed).  SMGX_EVENT_PATH=split selects the two-kernel path.
bool event_select_fused();
void set_event_select_fused(bool fused);
// 0 = pair (hash stream + search kernel), 1 = the warp-per-request family (simple / tiled / fused), 2 = one launch: hash stream whose last CTA per
// 256-request group runs the search (event_hs_kernel)
int event_path();
void set_event_path(int path);
void set_fused_minb(int minb);
void set_fused_prefetch(int pf);
void set_fused_tile(int tile, long long min_total);
void set_event_simple(int minb);
void set_tile_depth(int depth);
void launch_event_select(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream, uint64_t* launches);
// the two halves of the split path, for callers that pipeline them over two streams; event_launch_is_split: would launch_event_select run them?
bool event_launch_is_split(const MultiArgs& a);
void launch_event_hash(const MultiArgs& a, int sm_count, cudaStream_t stream, uint64_t* launches);
void launch_event_search(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream, uint64_t* launches);
// second phase of the load-feedback mode: one warp resolves a.total requests in order against running loads (starting from `loads`)
void launch_feedback_resolve(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, const uint64_t* d_loads, const uint8_t* d_flags,
                             uint32_t n_slice, uint64_t abs_threshold, float rel_threshold, uint64_t* d_loads_out, cudaStream_t stream);

// PositionalIndexer::find_matches on precomputed content hashes; one warp, one query.
void launch_find_matches(const EventIndexView& ix, const uint64_t* d_hashes, uint32_t n, bool early_exit, uint32_t* d_scores,
                         cudaStream_t stream);

// compute_request_content_hashes for one request.
void launch_content_hashes(const uint32_t* d_tokens, uint32_t n_tokens, uint32_t block_size, uint64_t* d_out, cudaStream_t stream);

void launch_content_hashes_ragged(const uint32_t* d_tokens, const uint32_t* d_offs, uint32_t n_blocks, uint64_t* d_out, cudaStream_t stream);
void launch_fill(uint32_t* d, uint32_t value, size_t n_words, cudaStream_t stream);
void launch_hold(uint32_t us, cudaStream_t stream);
// peer-memory exchange of the sharded pick (smgx.cu: Exchange)
void launch_shard_push(const smgx_shard_candidate* d_cand, uint32_t n, const smgx_shard_fleet* d_fleet, uint8_t* const* d_peer_parity_base, uint32_t world,
                       uint32_t rank, size_t cand_off, size_t cand_slot_bytes, size_t fleet_off, uint32_t fleet_stride, size_t flag_off, uint64_t seq,
                       uint32_t* d_arrive, cudaStream_t stream);
void launch_shard_reduce_wait(const uint8_t* d_parity_base, size_t cand_off, uint32_t cand_stride, size_t fleet_off, uint32_t fleet_stride, size_t flag_off,
                              uint64_t seq, const uint32_t* d_global_base, uint32_t world, uint32_t n, uint64_t abs_threshold, float rel_threshold,
                              int32_t* d_out_idx, smgx_decision_info* d_out_info, uint32_t* d_err, cudaStream_t stream);

// Merge of per-shard candidates (worker-id-sharded fleets): [world][n] candidates + [world] fleet summaries → picks.
void launch_shard_reduce(const smgx_shard_candidate* d_cands, const smgx_shard_fleet* d_fleets, const uint32_t* d_global_base, uint32_t world,
                         uint32_t n, uint64_t abs_threshold, float rel_threshold, int32_t* d_out_idx, smgx_decision_info* d_out_info,
                         cudaStream_t stream);

}  // namespace smgx
