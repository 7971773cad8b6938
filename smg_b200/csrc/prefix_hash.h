// Adjacent policy on the same plumbing (SURVEY §8f rank 4): `prefix_hash` (model_gateway/src/policies/prefix_hash.rs) over the
// consistent hash ring the registry hands to policies (model_gateway/src/worker/hash_ring.rs).  See prefix_hash.cu.
//
// Device layout per model:
//   ring_pos   [len] u64   sorted ring positions, len = 150 × ring URLs (hash_ring.rs:17, :45-70)
//   ring_slice [len] i32   per entry: LAST index of the worker slice whose url() equals the entry's URL, -1 = not in the slice
//   bucket     [2^k + 1] u32  radix index over the (uniformly distributed) positions, 2^k ≥ 2·len: replaces the binary search
//   ring_url   [len] u32   per entry: index into the ring's URL list (find_healthy_url with a caller-supplied predicate)
//   dup_prev   [n_slice] i32  previous slice index with the same URL (-1 = none): `healthy_url_map` is a HashMap collected from the
//                          healthy workers only, so the entry a URL resolves to is the last HEALTHY slice index with that URL (:155-159)
//   loads [n_slice] u64, flags [n_slice] u8 (bit0 = is_healthy()), derived (PrefixDerived, one per fleet snapshot)
#pragma once
#include <cstdint>

#include "common.h"

namespace smgx {

constexpr uint32_t kVirtualNodesPerWorker = 150;   // hash_ring.rs:17
constexpr int kMaxPrefixBatches = 32;

struct PrefixDerived {        // the per-call prologue of find_worker_with_load_balance (:137-149), once per fleet snapshot
    uint64_t total_load;      // Σ load() over healthy workers
    uint32_t n_healthy;
    int32_t least_ok;         // first argmin load() over healthy workers that pass load_ok (:176-179), -1 = none
    int32_t least_any;        // first argmin load() over healthy workers (:194-197)
    uint32_t all_ok;          // total_load == 0 || n_healthy == 0 (:117-119)
    double threshold;         // (total_load + 1) / n_healthy × load_factor, f64 (:122-124)
};

struct RingView {
    const uint64_t* pos; const int32_t* slice; uint32_t len; uint32_t has_ring;
    const uint32_t* bucket;     // [n_buckets + 1]: bucket[b] = partition_point(pos < (b << bucket_shift)); n_buckets = 2^k ≥ 2·len (≥ 2)
    uint32_t bucket_shift;      // 64 − k
};
struct PrefixFleetView { const uint64_t* loads; const uint8_t* flags; const int32_t* dup_prev; const PrefixDerived* derived; uint32_t n_slice; };

struct PrefixBatch {
    const uint32_t* tokens;       // device, ragged
    const uint32_t* offsets;      // device, n + 1
    const uint8_t* has_tokens;    // device, n; nullable (= every request carries Some(tokens))
    int32_t* out_idx;             // device, n; nullable
    smgx_decision_info* out_info; // device, n; nullable
    uint64_t* hash;               // device, n: compute_prefix_hash of each request (written by K-prefix-1, read by K-prefix-2)
    uint32_t n;
};
struct PrefixArgs { PrefixBatch b[kMaxPrefixBatches]; uint32_t count; uint32_t prefix_tokens; };

void launch_prefix_fleet_prepare(const uint64_t* d_loads, const uint8_t* d_flags, uint32_t n_slice, double load_factor, PrefixDerived* d_out, cudaStream_t stream);
// Load feedback: the picks of a launch are made in request order on running loads (prefix_candidate_kernel + prefix_feedback_kernel instead
// of prefix_pick_kernel).  run_loads (device, n_slice; nullable): the loads after the launch; from_run: start from them instead of the
// snapshot (the next launch of the same call continues the stream).  The fleet must fit in shared memory: kMaxFeedbackSlice.
struct PrefixFeedback { double load_factor; uint64_t* run_loads; uint32_t from_run; };
constexpr uint32_t kMaxFeedbackSlice = 200 * 1024 / 8;
// returns the number of kernels launched (1: hashes only, 2: hashes + picks, 3: hashes + the two load-feedback kernels)
// pick_stream == stream: all kernels in order on one stream; otherwise the pick kernels are ordered after `hashes_ready` on pick_stream
uint32_t launch_prefix_select(const RingView& ring, const PrefixFleetView& fleet, const PrefixArgs& a, cudaStream_t stream, cudaStream_t pick_stream,
                              cudaEvent_t hashes_ready, const PrefixFeedback* fb = nullptr);
// HashRing::find_healthy_url for precomputed key positions and a per-ring-URL predicate; out[i] = ring URL index or -1
void launch_ring_find(const uint64_t* d_ring_pos, const uint32_t* d_ring_url, uint32_t len, const uint64_t* d_key_pos, const uint8_t* d_url_ok, uint32_t n,
                      int32_t* d_out, cudaStream_t stream);

}  // namespace smgx
