// HashRing::find_healthy_url (worker/hash_ring.rs:102-134) from a key's ring position, over the healthy workers of the slice: the
// slice index the first ring URL at or clockwise after key_pos resolves to, -1 when no ring URL resolves to a healthy slice entry.
// Shared by prefix_hash (prefix_hash.cu) and consistent_hashing (consistent_hashing.cu); the ring must be non-empty.
#pragma once
#include <cstdint>

#include "prefix_hash.h"

namespace smgx {

__device__ __forceinline__ int32_t ring_walk(const RingView& ring, const PrefixFleetView& fleet, uint64_t key_pos) {
    int32_t initial = -1;
    // partition_point(|pos| pos < key_pos): positions are uniform 64-bit hashes, so a table of "first entry at or above
    // bucket b's lower bound" (2+ buckets per entry) lands within an entry or two of the answer — two dependent loads, not 14
    const uint32_t bk = (uint32_t)(key_pos >> ring.bucket_shift);
    uint32_t lo = __ldg(ring.bucket + bk);
    const uint32_t hi = __ldg(ring.bucket + bk + 1);
    while (lo < hi && __ldg(ring.pos + lo) < key_pos) ++lo;
    uint32_t e = lo == ring.len ? 0 : lo;
    for (uint32_t step = 0; step < ring.len; ++step) {
        int32_t s = __ldg(ring.slice + e);
        while (s >= 0 && !(fleet.flags[s] & 1)) s = fleet.dup_prev[s];   // the URL resolves to its last HEALTHY slice entry
        if (s >= 0) { initial = s; break; }
        if (++e == ring.len) e = 0;
    }
    return initial;
}

}  // namespace smgx
