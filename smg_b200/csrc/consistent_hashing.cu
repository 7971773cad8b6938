// consistent_hashing (policies/consistent_hashing.rs:116-186): header-based session affinity.
//
//   chash_kernel       one thread per request: header selection, HeaderValue::to_str (every byte \t or 0x20..=0x7E), the
//                      X-SMG-Target-Worker parse (usize::from_str), blake3 of a key of ≤ 1024 bytes (one chunk), the ring walk or the
//                      modulo fallback, and the random fallback.  A key of more than one chunk is queued instead.
//   chash_long_kernel  one warp per queued key, launched only when the batch holds a header value of more than 1024 bytes: lane j
//                      hashes chunk 32g + j of group g; the parent nodes are folded level by level (pairs (2k, 2k + 1), an odd last node
//                      carried up), which is blake3's "left subtree = largest power of two" tree.  Levels 1-5 stay inside a group of 32
//                      chunks (shuffles), the levels above run over the group values in shared memory.  Then the same decision.
// The healthy list and the URL → last healthy index list are derived once per fleet snapshot (Policy::sync_chash).
#include "consistent_hashing.h"

#include "blake3.cuh"
#include "common.h"
#include "counter_draw.cuh"
#include "ring_walk.cuh"

namespace smgx {
namespace {
using namespace b3;

constexpr int kThreads = 128;
constexpr int kLongWarps = 4;                                      // warps per CTA of the long-key kernel
constexpr uint32_t kMaxGroups = kChashMaxKeyBytes / (32u * 1024u);  // 32-chunk groups of the longest key

__device__ __forceinline__ bool visible_byte(uint32_t c) { return c == '\t' || c - 0x20u < 0x5Fu; }

// HeaderValue::to_str succeeds.  Cookies run to several KB, so the aligned middle is read as words, eight loads in flight per check.
__device__ __noinline__ bool visible_ascii(const uint8_t* __restrict__ p, uint32_t len) {
    uint32_t k = 0;
    bool ok = true;
    for (; k < len && (reinterpret_cast<uintptr_t>(p + k) & 3); ++k) ok &= visible_byte(__ldg(p + k));
    const uint32_t* w = reinterpret_cast<const uint32_t*>(p + k);
    const uint32_t nw = (len - k) / 4;
    for (uint32_t j = 0; j < nw && ok; j += 8) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            if (j + u < nw) {
                const uint32_t x = __ldg(w + j + u);
#pragma unroll
                for (int b = 0; b < 4; ++b) ok &= visible_byte((x >> (8 * b)) & 0xFFu);
            }
        }
    }
    for (k += 4 * nw; k < len; ++k) ok &= visible_byte(__ldg(p + k));
    return ok;
}

// `usize::from_str` (64-bit): an optional '+', then one or more ASCII digits, overflow is an error
__device__ __forceinline__ bool parse_usize(const uint8_t* __restrict__ p, uint32_t len, uint64_t& v) {
    uint32_t k = 0;
    if (len && __ldg(p) == '+') k = 1;
    if (k == len) return false;
    v = 0;
    for (; k < len; ++k) {
        const uint32_t d = (uint32_t)__ldg(p + k) - '0';
        if (d > 9) return false;
        if (v > (~0ull - d) / 10) return false;
        v = v * 10 + d;
    }
    return true;
}

// compress every block of one chunk of `len` ≤ 1024 bytes at p (counter = chunk index) into cv; `root` on the last block when the
// chunk is the whole input
__device__ __forceinline__ void chunk_cv(const uint8_t* __restrict__ p, uint32_t len, uint64_t counter, bool root, uint32_t cv[8]) {
#pragma unroll
    for (int q = 0; q < 8; ++q) cv[q] = kIV[q];
    const uint32_t n_blocks = len == 0 ? 1 : (len + 63) / 64;
    for (uint32_t b = 0; b < n_blocks; ++b) {
        const uint32_t blen = b + 1 == n_blocks ? len - 64 * b : 64;
        const uint8_t* bp = p + 64 * b;
        uint32_t m[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            uint32_t w = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) if ((uint32_t)(4 * q + k) < blen) w |= (uint32_t)__ldg(bp + 4 * q + k) << (8 * k);
            m[q] = w;
        }
        const uint32_t flags = (b == 0 ? CHUNK_START : 0u) | (b + 1 == n_blocks ? (CHUNK_END | (root ? ROOT : 0u)) : 0u);
        compress(cv, m, counter, blen, flags);
    }
}

__device__ __forceinline__ void parent_cv(uint32_t cv[8], const uint32_t right[8], bool root) {
    uint32_t m[16];
#pragma unroll
    for (int q = 0; q < 8; ++q) { m[q] = cv[q]; m[8 + q] = right[q]; cv[q] = kIV[q]; }
    compress(cv, m, 0, 64, PARENT | (root ? ROOT : 0u));
}

// find_by_consistent_hash (:68-111) from the key's ring position
__device__ __forceinline__ int32_t pick_by_key(const ChashArgs& a, uint64_t key_pos) {
    if (a.n_url_last == 0) return -1;                                                    // healthy_url_to_idx is empty (:80-82)
    if (a.ring.has_ring) return a.ring.len ? ring_walk(a.ring, a.fleet, key_pos) : -1;   // :85-89
    return __ldg(a.url_last + key_pos % a.n_url_last);                                   // sorted values, hash % len (:91-110)
}

__device__ __forceinline__ void write_out(const ChashArgs& a, uint32_t i, int32_t idx, uint8_t branch, uint64_t key_pos) {
    a.out_idx[i] = idx;
    a.out_branch[i] = branch;
    a.out_key_pos[i] = key_pos;
}

__global__ void __launch_bounds__(kThreads) chash_kernel(const ChashArgs a) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= a.n) return;
    if (a.fleet.n_slice == 0) { write_out(a, i, -1, SMGX_CH_NO_HEALTHY_WORKERS, 0); return; }   // :121-123
    const uint32_t* o = a.offsets + (size_t)kChashHeaders * i;
    const uint32_t present = __ldg(a.present + i);
    // extract_header_value: get(name) → to_str().ok() → non-empty (header_utils.rs:60-65)
    auto extracted = [&](uint32_t h) {
        const uint32_t b = __ldg(o + h), len = __ldg(o + h + 1) - b;
        return ((present >> h) & 1u) && len && visible_ascii(a.values + b, len);
    };
    if (extracted(0)) {                                                                   // X-SMG-Target-Worker (:128-137)
        const uint32_t b = __ldg(o), len = __ldg(o + 1) - b;
        uint64_t t;
        const bool hit = parse_usize(a.values + b, len, t) && t < a.fleet.n_slice && (a.fleet.flags[t] & 1);
        write_out(a, i, hit ? (int32_t)t : -1, hit ? SMGX_CH_TARGET_WORKER_HIT : SMGX_CH_TARGET_WORKER_MISS, 0);
        return;
    }
    int key = -1;
    if (extracted(1)) key = 1;                                                            // X-SMG-Routing-Key (:139-145)
    else {                                                                                // the first PRESENT of the three, then to_str (:147-155)
        const int h = (present & 4u) ? 2 : (present & 8u) ? 3 : (present & 16u) ? 4 : -1;
        if (h >= 0 && extracted((uint32_t)h)) key = h;
    }
    if (key >= 0) {
        const uint32_t b = __ldg(o + key), len = __ldg(o + key + 1) - b;
        if (len > 1024) {
            const uint32_t q = atomicAdd(a.queue_len, 1u);
            a.queue[q] = ChashLongKey{i, b, len};
            return;
        }
        uint32_t cv[8];
        chunk_cv(a.values + b, len, 0, true, cv);
        const uint64_t kp = ((uint64_t)cv[1] << 32) | cv[0];
        const int32_t idx = pick_by_key(a, kp);
        write_out(a, i, idx, idx >= 0 ? SMGX_CH_ROUTING_KEY_HIT : SMGX_CH_NO_HEALTHY_WORKERS, kp);
        return;
    }
    if (a.n_healthy == 0) { write_out(a, i, -1, SMGX_CH_NO_HEALTHY_WORKERS, 0); return; }   // :164-167
    const uint32_t r = (uint32_t)__umul64hi(p2c_draw(a.seed, i), (uint64_t)a.n_healthy);     // random_range(0..healthy_count) (:169-176)
    write_out(a, i, __ldg(a.healthy + r), SMGX_CH_RANDOM_FALLBACK, 0);
}

__global__ void __launch_bounds__(32 * kLongWarps) chash_long_kernel(const ChashArgs a) {
    __shared__ uint32_t s_cv[kLongWarps][kMaxGroups][8];
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t count = *a.queue_len;
    for (uint32_t q = blockIdx.x * kLongWarps + w; q < count; q += gridDim.x * kLongWarps) {
        const ChashLongKey k = a.queue[q];
        const uint8_t* p = a.values + k.start;
        const uint32_t n_chunks = (k.len + 1023) / 1024, n_groups = (n_chunks + 31) / 32;   // n_chunks ≥ 2
        uint32_t cv[8];
        for (uint32_t g = 0; g < n_groups; ++g) {
            const uint32_t c = 32 * g + lane, in_group = min(32u, n_chunks - 32 * g);
            if (c < n_chunks) chunk_cv(p + 1024ull * c, min(1024u, k.len - 1024 * c), c, false, cv);
            // levels 1-5: node j of a level sits in lane j·s; the last merge of a single-group key is the root
            for (uint32_t s = 1, cnt = in_group; cnt > 1; s <<= 1, cnt = (cnt + 1) / 2) {
                uint32_t right[8];
#pragma unroll
                for (int x = 0; x < 8; ++x) right[x] = __shfl_down_sync(0xFFFFFFFFu, cv[x], s);
                if ((lane & (2 * s - 1)) == 0 && lane / s + 1 < cnt) parent_cv(cv, right, n_groups == 1 && cnt == 2);
            }
            if (lane == 0 && n_groups > 1) {
#pragma unroll
                for (int x = 0; x < 8; ++x) s_cv[w][g][x] = cv[x];
            }
        }
        if (n_groups > 1) {   // levels 6+: pairs of group values, the last merge is the root
            __syncwarp();
            for (uint32_t cnt = n_groups; cnt > 1; cnt = (cnt + 1) / 2) {
                const uint32_t half = cnt / 2;   // ≤ 32
                if (lane < half) {
#pragma unroll
                    for (int x = 0; x < 8; ++x) { cv[x] = s_cv[w][2 * lane][x]; }
                    uint32_t right[8];
#pragma unroll
                    for (int x = 0; x < 8; ++x) right[x] = s_cv[w][2 * lane + 1][x];
                    parent_cv(cv, right, cnt == 2);
                }
                uint32_t carry[8];
#pragma unroll
                for (int x = 0; x < 8; ++x) carry[x] = s_cv[w][cnt - 1][x];
                __syncwarp();
                if (lane < half) {
#pragma unroll
                    for (int x = 0; x < 8; ++x) s_cv[w][lane][x] = cv[x];
                }
                if (lane == 0 && (cnt & 1)) {
#pragma unroll
                    for (int x = 0; x < 8; ++x) s_cv[w][half][x] = carry[x];
                }
                __syncwarp();
            }
        }
        if (lane == 0) {
            const uint64_t kp = ((uint64_t)cv[1] << 32) | cv[0];
            const int32_t idx = pick_by_key(a, kp);
            write_out(a, k.req, idx, idx >= 0 ? SMGX_CH_ROUTING_KEY_HIT : SMGX_CH_NO_HEALTHY_WORKERS, kp);
        }
        __syncwarp();
    }
}

}  // namespace

uint32_t launch_consistent_hashing(const ChashArgs& a, uint32_t max_long, int sm_count, cudaStream_t stream) {
    if (!a.n) return 0;
    if (max_long) SMGX_CUDA(cudaMemsetAsync(a.queue_len, 0, 4, stream));
    chash_kernel<<<(a.n + kThreads - 1) / kThreads, kThreads, 0, stream>>>(a);
    if (max_long) {
        const uint32_t ctas = std::min<uint32_t>((max_long + kLongWarps - 1) / kLongWarps, (uint32_t)std::max(sm_count, 1) * 8);
        chash_long_kernel<<<ctas, 32 * kLongWarps, 0, stream>>>(a);
    }
    SMGX_CUDA(cudaGetLastError());
    return max_long ? 2u : 1u;
}

}  // namespace smgx
