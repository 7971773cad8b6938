// consistent_hashing policy (model_gateway/src/policies/consistent_hashing.rs:116-186) for a batch of requests: one thread per request,
// plus one warp per routing key longer than one blake3 chunk.  See consistent_hashing.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "prefix_hash.h"

namespace smgx {

constexpr uint32_t kChashHeaders = 5;              // x-smg-target-worker, x-smg-routing-key, authorization, x-forwarded-for, cookie
constexpr uint32_t kChashMaxKeyBytes = 2u << 20;   // longest key value the long-key path hashes: 64 groups of 32 chunks

struct ChashLongKey { uint32_t req, start, len; };   // a key of > 1024 bytes, queued by the per-request kernel

struct ChashArgs {
    const uint8_t* values;      // device: header bytes of the batch
    const uint32_t* offsets;    // device [5n + 1]: header h of request i = values[offsets[5i + h] .. offsets[5i + h + 1])
    const uint8_t* present;     // device [n]: bit h = HeaderMap::get(name h) returned Some
    uint32_t n;
    uint64_t seed;              // random fallback: request i uses draw i of this stream
    RingView ring;              // has_ring = 0 ⇔ info.hash_ring is None
    PrefixFleetView fleet;      // flags bit 0 = is_healthy(), dup_prev, n_slice (loads and derived are not read)
    const int32_t* healthy;     // device [n_healthy]: ascending slice indices of the is_healthy() workers (random fallback)
    uint32_t n_healthy;
    const int32_t* url_last;    // device [n_url_last]: ascending values of the healthy URL → last healthy slice index map (modulo fallback)
    uint32_t n_url_last;
    int32_t* out_idx;           // device [n]: slice index, -1 = None
    uint8_t* out_branch;        // device [n]: smgx_ch_branch
    uint64_t* out_key_pos;      // device [n]: blake3(key)[..8] LE of the key used, 0 when none
    ChashLongKey* queue;        // device [n]: keys for the long-key kernel
    uint32_t* queue_len;        // device: zeroed before the per-request kernel when max_long != 0
};

// max_long: upper bound on the keys longer than 1024 bytes (0: the long-key kernel is not launched).  Returns the kernels launched.
uint32_t launch_consistent_hashing(const ChashArgs& a, uint32_t max_long, int sm_count, cudaStream_t stream);

}  // namespace smgx
