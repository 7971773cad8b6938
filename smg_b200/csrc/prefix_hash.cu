// prefix_hash policy on the GPU (model_gateway/src/policies/prefix_hash.rs:106-222) — two launches per batch (or per ≤ 32 batches):
//
//   K-prefix-1  compute_prefix_hash (:106-113): XXH3-64 (seed 0) of the first min(n, prefix_token_count) tokens, EIGHT LANES PER REQUEST
//            (lane i owns XXH3's accumulator i; see xxh3_group), four requests per warp.
//            This is the only HBM traffic of the policy: ≤ prefix_token_count × 4 bytes per request, read once.
//   K-prefix-2  one thread per request: format!("{prefix_hash:016x}") → blake3 of those 16 bytes (one compression, hash_ring.rs:78-86)
//            → partition_point over the sorted ring (:110) → clockwise walk to the first healthy worker of the slice (:119-131)
//            → load_ok / least-loaded fallback against the fleet summary computed once per snapshot (prefix_hash.rs:116-127, :164-197).
//            Ring (150 entries per worker) and fleet arrays are a few hundred KB and stay in L2.
#include "prefix_hash.h"

#include "blake3.cuh"
#include "ring_walk.cuh"
#include "xxh3.cuh"

namespace smgx {
namespace {

constexpr int kThreads = 128;       // pick kernel: one thread per request
constexpr int kHashThreads = 64;    // hash kernel: 2 warps × 4 requests, one round — short CTAs keep the last wave of a launch small (32 and 128 threads measured slower)
constexpr int kWarps = kHashThreads / 32;
constexpr int kReqPerCta = kWarps * 4;

// inputs of ≤ 240 bytes take XXH3's short forms: a handful of dependent multiplies, done by every lane on the same words
__device__ __noinline__ uint64_t xxh3_small(const uint32_t* __restrict__ w, uint32_t n) { return xxh3_words_upto60(w, n, 0); }

// ---- XXH3-64 (seed 0) of n > 60 words by a group of 8 lanes: lane i owns accumulator i for every stripe ----
// Above 240 bytes XXH3 folds 64-byte stripes into eight 64-bit accumulators; accumulator i of a stripe needs data qword i (multiply)
// and qword i ^ 1 (add).  Lane i of the group therefore reads qword i of every stripe (the group reads one whole stripe, 64 contiguous
// bytes, per instruction), keeps acc[i] and the running sum of its own data, and hands that sum to lane i ^ 1 once per 1 KiB block.
// Four requests share a warp, so every load / xor / multiply instruction serves four requests and the fixed tail (merge + avalanche)
// is paid once per four.
struct GroupKeys {
    uint64_t last;             // last stripe: secret bytes 121 + 8·i
    uint64_t scramble;         // secret bytes 128 + 8·i
    uint64_t merge0, merge1;   // final merge of accumulators (2j, 2j+1), j = i & 3: secret bytes 11 + 16·j, +8
    uint64_t init;             // initial accumulator i
};

__device__ __forceinline__ GroupKeys group_keys(int i) {
    GroupKeys k;
    k.last = sec64_unaligned(121 + 8 * i);
    k.scramble = sec64(128 + 8 * i);
    k.merge0 = sec64_unaligned(11 + 16 * (i & 3));
    k.merge1 = sec64_unaligned(19 + 16 * (i & 3));
    const uint64_t init[8] = {P32_3, P64_1, P64_2, P64_3, P64_4, P32_2, P64_5, P32_1};
    k.init = init[0];
#pragma unroll
    for (int q = 1; q < 8; ++q) if (i == q) k.init = init[q];
    return k;
}

template <bool kAligned>
__device__ __forceinline__ uint64_t ldq(const uint32_t* __restrict__ p) {
    if (kAligned) { const uint2 v = __ldg(reinterpret_cast<const uint2*>(p)); return mk64(v.x, v.y); }
    return mk64(__ldg(p), __ldg(p + 1));
}

// s_sec: the default secret as 24 qwords in shared memory (stripe s, accumulator i reads qword s + i)
template <bool kAligned>
__device__ __forceinline__ uint64_t xxh3_group(const uint32_t* __restrict__ w, uint32_t n, int i, uint32_t gmask, const GroupKeys& k,
                                               const uint64_t* __restrict__ s_sec) {
    const uint32_t len = n * 4;
    const uint32_t nb_blocks = (len - 1) >> 10;
    uint64_t acc = k.init;
    const uint32_t* p = w + 2 * i;
    for (uint32_t b = 0; b < nb_blocks; ++b, p += 256) {
        uint64_t A = 0, B = 0;
#pragma unroll
        for (int st = 0; st < 16; ++st) {
            const uint64_t dv = ldq<kAligned>(p + st * 16), dk = dv ^ s_sec[st + i];
            A += (dk & 0xFFFFFFFFULL) * (dk >> 32);
            B += dv;
        }
        acc += A + __shfl_xor_sync(gmask, B, 1);
        acc = (acc ^ (acc >> 47) ^ k.scramble) * P32_1;
    }
    const uint32_t nst = ((len - 1) - (nb_blocks << 10)) >> 6;   // whole stripes of the last, partial block (0..15)
    // all sixteen loads first: 4 KB per warp in flight
    uint64_t A = 0, B = 0;
    const uint32_t* lw = w + n - 16 + 2 * i;
    const bool last_al = (reinterpret_cast<uintptr_t>(lw) & 7) == 0;
    uint64_t d[16];
#pragma unroll
    for (int st = 0; st < 15; ++st) d[st] = (uint32_t)st < nst ? ldq<kAligned>(p + st * 16) : 0;
    d[15] = last_al ? ldq<true>(lw) : ldq<false>(lw);   // the last 64 bytes of the input, against secret bytes [121, 185)
#pragma unroll
    for (int st = 0; st < 15; ++st) {
        if ((uint32_t)st < nst) {
            const uint64_t dk = d[st] ^ s_sec[st + i];
            A += (dk & 0xFFFFFFFFULL) * (dk >> 32);
            B += d[st];
        }
    }
    {
        const uint64_t dk = d[15] ^ k.last;
        A += (dk & 0xFFFFFFFFULL) * (dk >> 32);
        B += d[15];
    }
    acc += A + __shfl_xor_sync(gmask, B, 1);
    // merge: len·P64_1 + Σ_j mul128_fold64(acc[2j] ^ k0_j, acc[2j+1] ^ k1_j); lane j = i & 3 takes pair j
    const int lane = threadIdx.x & 31, base = lane & ~7, j = i & 3;
    const uint64_t a0 = __shfl_sync(gmask, acc, base + 2 * j), a1 = __shfl_sync(gmask, acc, base + 2 * j + 1);
    uint64_t r = mul128_fold64(a0 ^ k.merge0, a1 ^ k.merge1);
    r += __shfl_xor_sync(gmask, r, 1);
    r += __shfl_xor_sync(gmask, r, 2);
    return avalanche((uint64_t)len * P64_1 + r);
}

__device__ __forceinline__ bool load_ok(uint64_t load, const PrefixDerived& d) {   // prefix_hash.rs:116-127
    return d.all_ok || (double)load <= d.threshold;
}

// K-prefix-1: compute_prefix_hash of every request → bt.hash[r].  8 lanes per request, 4 requests per warp, kRounds (= 1) rounds per warp.
__global__ void __launch_bounds__(kHashThreads) prefix_hash_kernel(const __grid_constant__ PrefixArgs a) {
    const PrefixBatch& bt = a.b[blockIdx.y];
    const uint32_t first = blockIdx.x * kReqPerCta;
    if (first >= bt.n) return;
    __shared__ uint64_t s_sec[24];
    if (threadIdx.x < 24) s_sec[threadIdx.x] = sec64(8 * threadIdx.x);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane >> 3, i = lane & 7;
    const uint32_t gmask = 0xFFu << (8 * sub);
    const GroupKeys keys = group_keys(i);
    constexpr int kRounds = kReqPerCta / (kWarps * 4);
#pragma unroll 1
    for (int round = 0; round < kRounds; ++round) {
        const uint32_t r = first + (warp * kRounds + round) * 4 + sub;
        const bool valid = r < bt.n;
        uint32_t beg = 0, n = 0;
        if (valid) { beg = __ldg(bt.offsets + r); n = __ldg(bt.offsets + r + 1) - beg; }
        const uint32_t use = min(n, a.prefix_tokens);
        const uint32_t* w = bt.tokens + beg;
        const bool al = (reinterpret_cast<uintptr_t>(w) & 7) == 0;
        const bool all_al = __all_sync(0xFFFFFFFFu, al || !valid || use <= 60);
        if (!valid) continue;
        uint64_t h;
        if (use <= 60) h = xxh3_small(w, use);
        else if (all_al) h = xxh3_group<true>(w, use, i, gmask, keys, s_sec);
        else h = xxh3_group<false>(w, use, i, gmask, keys, s_sec);
        if (i == 0) bt.hash[r] = h;
    }
}

// HashRing::find_healthy_url (hash_ring.rs:102-134) of a request's prefix hash over the slice's healthy workers: its ring candidate,
// -1 when no ring URL resolves to a healthy slice entry.  Shared by the pick kernel and the load-feedback candidate kernel.
__device__ __forceinline__ int32_t ring_candidate(const RingView& ring, const PrefixFleetView& fleet, uint64_t ph) {
    // key = format!("{prefix_hash:016x}"): 16 lower-case hex digits, most significant first, as one blake3 block
    uint32_t m[16];
#pragma unroll
    for (int wd = 0; wd < 4; ++wd) {
        uint32_t word = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const uint32_t nib = (uint32_t)(ph >> (60 - 4 * (4 * wd + c))) & 15u;
            word |= (nib < 10 ? '0' + nib : 'a' + nib - 10) << (8 * c);
        }
        m[wd] = word;
    }
#pragma unroll
    for (int wd = 4; wd < 16; ++wd) m[wd] = 0;
    uint32_t cv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) cv[q] = b3::kIV[q];
    b3::compress(cv, m, 0, 16, b3::CHUNK_START | b3::CHUNK_END | b3::ROOT);
    return ring_walk(ring, fleet, mk64(cv[0], cv[1]));
}

// K-prefix-2: one thread per request: ring lookup + bounded-load pick from bt.hash[r]
__global__ void __launch_bounds__(kThreads) prefix_pick_kernel(const RingView ring, const PrefixFleetView fleet, const __grid_constant__ PrefixArgs a) {
    const PrefixBatch& bt = a.b[blockIdx.y];
    const uint32_t r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= bt.n || !bt.out_idx) return;
    const uint64_t ph = bt.hash[r];
    const uint32_t n_tok = __ldg(bt.offsets + r + 1) - __ldg(bt.offsets + r);
    const PrefixDerived d = *fleet.derived;
    int32_t idx = -1;
    uint8_t branch;
    const bool some = n_tok != 0 && (bt.has_tokens == nullptr || bt.has_tokens[r] != 0);
    if (fleet.n_slice == 0) branch = SMGX_PH_NO_HEALTHY_WORKERS;        // workers.is_empty() (:208-210)
    else if (!some) branch = SMGX_PH_NO_TOKENS;                         // :213-216
    else if (d.n_healthy == 0) branch = SMGX_PH_NO_HEALTHY_WORKERS;     // :143-145
    else {
        const int32_t initial = (ring.has_ring && ring.len) ? ring_candidate(ring, fleet, ph) : -1;
        if (initial >= 0) {
            if (load_ok(fleet.loads[initial], d)) { idx = initial; branch = SMGX_PH_RING_HIT; }
            else { idx = d.least_ok >= 0 ? d.least_ok : initial; branch = SMGX_PH_LOAD_BALANCE_WALK; }
        } else { idx = d.least_any; branch = SMGX_PH_FALLBACK_LEAST_LOAD; }
    }
    bt.out_idx[r] = idx;
    if (bt.out_info) {
        smgx_decision_info o;
        o.matched = 0; o.input = n_tok; o.branch = branch; o.nodes = 0; o.reserved[0] = o.reserved[1] = 0;
        bt.out_info[r] = o;
    }
}

// (load, idx) lexicographic minimum = Iterator::min_by_key's FIRST minimum
__device__ __forceinline__ void take_min(uint64_t& load, int32_t& idx, uint64_t ol, int32_t oi) {
    if (oi >= 0 && (idx < 0 || ol < load || (ol == load && oi < idx))) { load = ol; idx = oi; }
}

// ---- load feedback (smgx_set_load_feedback_policies, SMGX_FEEDBACK_PREFIX_HASH): the batch as the request stream of a router that guards
// every pick (routers/grpc/context.rs:248-259), request i seeing the snapshot loads plus one per pick of requests < i ----
constexpr int64_t kPhNoRing = -1;     // no ring, or no ring URL resolves to a healthy slice entry → least loaded healthy worker
constexpr int64_t kPhDecided = -2;    // None (no worker, no tokens, no healthy worker): written by the candidate kernel

// phase 1, one thread per request: everything prefix_pick_kernel decides without loads.  bt.hash[r] is replaced by the request's ring
// candidate, kPhNoRing or kPhDecided.
__global__ void __launch_bounds__(kThreads) prefix_candidate_kernel(const RingView ring, const PrefixFleetView fleet, const __grid_constant__ PrefixArgs a) {
    const PrefixBatch& bt = a.b[blockIdx.y];
    const uint32_t r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= bt.n || !bt.out_idx) return;
    const uint64_t ph = bt.hash[r];
    const uint32_t n_tok = __ldg(bt.offsets + r + 1) - __ldg(bt.offsets + r);
    const bool some = n_tok != 0 && (bt.has_tokens == nullptr || bt.has_tokens[r] != 0);
    int64_t cand = kPhDecided;
    uint8_t branch = SMGX_PH_NO_HEALTHY_WORKERS;
    if (fleet.n_slice == 0) branch = SMGX_PH_NO_HEALTHY_WORKERS;             // :208-210
    else if (!some) branch = SMGX_PH_NO_TOKENS;                              // :213-216
    else if (fleet.derived->n_healthy != 0) cand = (ring.has_ring && ring.len) ? ring_candidate(ring, fleet, ph) : kPhNoRing;   // else :143-145
    bt.hash[r] = (uint64_t)cand;
    if (cand != kPhDecided) return;
    bt.out_idx[r] = -1;
    if (bt.out_info) {
        smgx_decision_info o;
        o.matched = 0; o.input = n_tok; o.branch = branch; o.nodes = 0; o.reserved[0] = o.reserved[1] = 0;
        bt.out_info[r] = o;
    }
}

// phase 2, one warp, the requests of every batch of the launch in order: running loads in shared memory, the running Σ load() over healthy
// workers and the threshold (Σ + 1) as f64 / n × load_factor in the operation order of prefix_fleet_prepare_kernel, the first healthy argmin
// (looked for again only after it was picked).  load_ok is monotone in the load, so "least loaded worker passing load_ok" is that argmin when
// it passes and none otherwise.  Loads start from `run` when from_run (a previous launch of the same call) and are left in `run` if non-null.
__global__ void __launch_bounds__(32) prefix_feedback_kernel(const PrefixFleetView fleet, const __grid_constant__ PrefixArgs a, double load_factor,
                                                             uint64_t* __restrict__ run, uint32_t from_run) {
    extern __shared__ uint64_t s_L[];   // [n_slice]
    const int lane = threadIdx.x;
    const uint32_t ns = fleet.n_slice;
    uint64_t total = 0;
    for (uint32_t i = lane; i < ns; i += 32) {
        const uint64_t l = from_run ? run[i] : fleet.loads[i];
        s_L[i] = l;
        if (fleet.flags[i] & 1) total += l;
    }
    for (int m = 16; m; m >>= 1) total += __shfl_xor_sync(0xFFFFFFFFu, total, m);
    __syncwarp();
    const uint32_t nh = fleet.derived->n_healthy;
    auto least = [&]() {   // first argmin load over healthy workers (min_by_key → FIRST minimum)
        uint64_t bl = 0; int32_t bi = -1;
        for (uint32_t i = lane; i < ns; i += 32) if (fleet.flags[i] & 1) take_min(bl, bi, s_L[i], (int32_t)i);
        for (int m = 16; m; m >>= 1) {
            const uint64_t ol = __shfl_xor_sync(0xFFFFFFFFu, bl, m);
            const int32_t oi = __shfl_xor_sync(0xFFFFFFFFu, bi, m);
            take_min(bl, bi, ol, oi);
        }
        return bi;
    };
    int32_t hidx = least();
    for (uint32_t j = 0; j < a.count; ++j) {
        const PrefixBatch& bt = a.b[j];
        if (!bt.out_idx) continue;
        for (uint32_t r = 0; r < bt.n; ++r) {
            const int64_t cand = (int64_t)bt.hash[r];
            if (cand == kPhDecided) continue;
            const bool all_ok = total == 0 || nh == 0;                                   // :117-119
            const double thr = nh ? __dmul_rn(__ddiv_rn((double)(total + 1), (double)nh), load_factor) : 0.0;
            int32_t idx;
            uint8_t branch;
            if (cand >= 0) {
                const int32_t c = (int32_t)cand;
                if (all_ok || (double)s_L[c] <= thr) { idx = c; branch = SMGX_PH_RING_HIT; }
                else { idx = (hidx >= 0 && (double)s_L[hidx] <= thr) ? hidx : c; branch = SMGX_PH_LOAD_BALANCE_WALK; }
            } else { idx = hidx; branch = SMGX_PH_FALLBACK_LEAST_LOAD; }
            if (lane == 0) {
                bt.out_idx[r] = idx;
                if (bt.out_info) {
                    smgx_decision_info o;
                    o.matched = 0; o.input = __ldg(bt.offsets + r + 1) - __ldg(bt.offsets + r); o.branch = branch; o.nodes = 0;
                    o.reserved[0] = o.reserved[1] = 0;
                    bt.out_info[r] = o;
                }
            }
            if (idx < 0) continue;
            const uint64_t old = s_L[idx];   // the guard: load() + 1 on the pick (a healthy worker, so Σ grows too)
            __syncwarp();
            if (lane == 0) s_L[idx] = old + 1;
            __syncwarp();
            total += 1;
            if (idx == hidx) hidx = least();
        }
    }
    if (run) for (uint32_t i = lane; i < ns; i += 32) run[i] = s_L[i];
}

__global__ void __launch_bounds__(256) prefix_fleet_prepare_kernel(const uint64_t* __restrict__ loads, const uint8_t* __restrict__ flags, uint32_t n_slice,
                                                                   double load_factor, PrefixDerived* __restrict__ out) {
    __shared__ uint64_t s_total[8], s_load[8];
    __shared__ uint32_t s_cnt[8];
    __shared__ int32_t s_idx[8];
    __shared__ PrefixDerived s_d;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t total = 0;
    uint32_t cnt = 0;
    for (uint32_t i = threadIdx.x; i < n_slice; i += blockDim.x)
        if (flags[i] & 1) { total += loads[i]; ++cnt; }
    for (int m = 16; m; m >>= 1) { total += __shfl_xor_sync(0xFFFFFFFFu, total, m); cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, m); }
    if (lane == 0) { s_total[warp] = total; s_cnt[warp] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t t = 0; uint32_t c = 0;
        for (int w = 0; w < 8; ++w) { t += s_total[w]; c += s_cnt[w]; }
        s_d.total_load = t; s_d.n_healthy = c;
        s_d.all_ok = (t == 0 || c == 0) ? 1u : 0u;
        // avg_load = (total_load + 1) as f64 / num_workers as f64; threshold = avg_load * load_factor  (:122-124)
        s_d.threshold = c ? __dmul_rn(__ddiv_rn((double)(t + 1), (double)c), load_factor) : 0.0;
    }
    __syncthreads();
    const PrefixDerived d = s_d;
    for (int pass = 0; pass < 2; ++pass) {   // 0: least loaded among those passing load_ok, 1: least loaded healthy
        uint64_t bl = 0; int32_t bi = -1;
        for (uint32_t i = threadIdx.x; i < n_slice; i += blockDim.x)
            if ((flags[i] & 1) && (pass == 1 || load_ok(loads[i], d))) take_min(bl, bi, loads[i], (int32_t)i);
        for (int m = 16; m; m >>= 1) {
            const uint64_t ol = __shfl_xor_sync(0xFFFFFFFFu, bl, m);
            const int32_t oi = __shfl_xor_sync(0xFFFFFFFFu, bi, m);
            take_min(bl, bi, ol, oi);
        }
        if (lane == 0) { s_load[warp] = bl; s_idx[warp] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint64_t l = 0; int32_t x = -1;
            for (int w = 0; w < 8; ++w) take_min(l, x, s_load[w], s_idx[w]);
            if (pass == 0) s_d.least_ok = x; else s_d.least_any = x;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = s_d;
}

__global__ void __launch_bounds__(128) ring_find_kernel(const uint64_t* __restrict__ ring_pos, const uint32_t* __restrict__ ring_url, uint32_t len,
                                                        const uint64_t* __restrict__ key_pos, const uint8_t* __restrict__ url_ok, uint32_t n,
                                                        int32_t* __restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    int32_t found = -1;
    if (len) {
        const uint64_t kp = key_pos[t];
        uint32_t lo = 0, hi = len;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (ring_pos[mid] < kp) lo = mid + 1; else hi = mid; }
        uint32_t e = lo == len ? 0 : lo;
        for (uint32_t step = 0; step < len; ++step) {
            const uint32_t u = ring_url[e];
            if (url_ok[u]) { found = (int32_t)u; break; }
            if (++e == len) e = 0;
        }
    }
    out[t] = found;
}

}  // namespace

void launch_prefix_fleet_prepare(const uint64_t* d_loads, const uint8_t* d_flags, uint32_t n_slice, double load_factor, PrefixDerived* d_out, cudaStream_t stream) {
    prefix_fleet_prepare_kernel<<<1, 256, 0, stream>>>(d_loads, d_flags, n_slice, load_factor, d_out);
    SMGX_CUDA(cudaGetLastError());
}

uint32_t launch_prefix_select(const RingView& ring, const PrefixFleetView& fleet, const PrefixArgs& a, cudaStream_t stream, cudaStream_t pick_stream,
                              cudaEvent_t hashes_ready, const PrefixFeedback* fb) {
    uint32_t max_n = 0;
    for (uint32_t k = 0; k < a.count; ++k) max_n = max_n > a.b[k].n ? max_n : a.b[k].n;
    if (max_n == 0 || a.count == 0) return 0;
    prefix_hash_kernel<<<dim3((max_n + kReqPerCta - 1) / kReqPerCta, a.count), kHashThreads, 0, stream>>>(a);
    bool pick = false;
    for (uint32_t k = 0; k < a.count; ++k) pick = pick || a.b[k].out_idx != nullptr;
    if (pick) {
        if (pick_stream != stream) {   // the latency-bound pick runs beside the next group's bandwidth-bound hash kernel
            SMGX_CUDA(cudaEventRecord(hashes_ready, stream));
            SMGX_CUDA(cudaStreamWaitEvent(pick_stream, hashes_ready, 0));
        }
        if (!fb) prefix_pick_kernel<<<dim3((max_n + kThreads - 1) / kThreads, a.count), kThreads, 0, pick_stream>>>(ring, fleet, a);
        else {
            const size_t smem = (size_t)(fleet.n_slice ? fleet.n_slice : 1) * 8;
            if (smem > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(prefix_feedback_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            prefix_candidate_kernel<<<dim3((max_n + kThreads - 1) / kThreads, a.count), kThreads, 0, pick_stream>>>(ring, fleet, a);
            prefix_feedback_kernel<<<1, 32, smem, pick_stream>>>(fleet, a, fb->load_factor, fb->run_loads, fb->from_run);
        }
    }
    SMGX_CUDA(cudaGetLastError());
    return pick ? (fb ? 3u : 2u) : 1u;
}

void launch_ring_find(const uint64_t* d_ring_pos, const uint32_t* d_ring_url, uint32_t len, const uint64_t* d_key_pos, const uint8_t* d_url_ok, uint32_t n,
                      int32_t* d_out, cudaStream_t stream) {
    if (n == 0) return;
    ring_find_kernel<<<(n + 127) / 128, 128, 0, stream>>>(d_ring_pos, d_ring_url, len, d_key_pos, d_url_ok, n, d_out);
    SMGX_CUDA(cudaGetLastError());
}

}  // namespace smgx
