// sm_90a kernels for the event-driven cache-aware pick.
//
//   K2b  content hashes (XXH3-64, seed 1337) of every full block of a request
//          ← compute_request_content_hashes      crates/kv_index/src/event_tree.rs:141-151
//        jump search over the GPU-resident positional index, exact reference semantics incl. the count-only
//        jump test, the retain guard and Single/Multi entries
//          ← PositionalIndexer::jump_search_matches / linear_scan_drain / count_workers_at  event_tree.rs:555-753
//   K3   per-worker (overlap, load, tree_size) → argmax worker with the reference's tie-breaks, min-load fallback
//          ← CacheAwarePolicy::score_overlap / select_worker_event_driven   cache_aware.rs:736-831
//        fleet_prepare: healthy filter, min/max load, f32 imbalance gate, first-min-load
//          ← select_worker prologue   cache_aware.rs:651-670, policies/mod.rs:137-144
//
// What runs by default (launch_event_select, bottom of the file): the PAIR — hash_blocks_kernel (one thread per 64 B block, a pure HBM
// stream; writes hash rows + one record per request, prefetches the first two index slots evict-last while the tokens are loaded
// evict-first) followed by event_search2_kernel as a programmatic dependent launch (≤ 64 interned workers; one thread per request, then
// balanced drains) or event_search_warp_kernel (wider fleets: one warp per request, one u64 set word per lane).  Mapped submissions and
// load-feedback batches run event_fused_kernel (+ feedback_resolve_kernel).
//
// Contents, in file order:
//   shared device code     slot probes, worker-set algebra, scan_drain / jump_search (generic search), hash_block
//   hash_blocks_kernel     the hash stream
//   event_search_thread_kernel, event_search_warp_kernel
//   finish_pick, drain_resolve   argmax + store of one request; the register drain of a failed count test (search2 and the warp kernel)
//   search2_body / event_search2_kernel
//   alternatives           (SMGX_EVENT_PATH, every one parity-green; on H100 event_lane_kernel below is the default, the pair is `split`)
//       event_hs_kernel        hash stream whose last CTA per 256-request group searches
//       event_stream_kernel    persistent, warp-specialised, fed by bulk async copies (+ stream_search)
//       event_tile_kernel      one warp per 8 / 16 / 32 requests
//       event_lane_kernel      one thread per request, failed count tests drained across the CTA, event_slow_kernel for rare shapes
//       event_warp_kernel      the same pick, one warp per request, for launches of fewer than 256 requests per SM
//       event_fused_kernel     persistent warp per request (also the mapped / feedback path)
//   small kernels          find_matches, content_hashes, fill, fleet_prepare
//   launchers              path selection (event_path), launch_event_hash / _search / _select
//   feedback_resolve_kernel, shard_push / shard_reduce kernels (sharded fleets), hold_kernel (gated timing)
// No tensor-core work exists on this path: it is integer hashing and 32 B probes, HBM-bound.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <string>

#include "kernels.h"
#include "xxh3.cuh"

namespace smgx {
namespace {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(FULL, (uint32_t)v, src), hi = __shfl_sync(FULL, (uint32_t)(v >> 32), src);
    return mk64(lo, hi);
}
__device__ __forceinline__ uint64_t shfl64_xor(uint64_t v, int m) {
    uint32_t lo = __shfl_xor_sync(FULL, (uint32_t)v, m), hi = __shfl_xor_sync(FULL, (uint32_t)(v >> 32), m);
    return mk64(lo, hi);
}

__device__ __forceinline__ Slot load_slot(const Slot* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    Slot s;
    s.content = mk64(a.x, a.y); s.pos = a.z; s.state = a.w;
    s.run = b.x; s.pad = b.y; s.payload = mk64(b.z, b.w);
    return s;
}
__device__ __forceinline__ MultiNode load_node(const MultiNode* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    MultiNode n;
    n.prefix = mk64(a.x, a.y); n.payload = mk64(a.z, a.w); n.next = b.x; n.pad0 = 0; n.pad1 = 0;
    return n;
}

// 16 B of the tag array, kept in L2 (evict-last): the tags are 1/32 of the slots' size and are read by every chain walk
__device__ __forceinline__ uint4 ld_tags(const uint8_t* p) {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    uint4 r;
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
// bit k set ⟺ byte k of the 16 B word equals the byte replicated in `rep`
__device__ __forceinline__ uint32_t byte_eq_bits(const uint4 w, uint32_t rep) {
    auto four = [&](uint32_t x) { return ((__vcmpeq4(x, rep) & 0x01010101u) * 0x01020408u) >> 24; };   // bytes 0..3 → bits 0..3
    return four(w.x) | (four(w.y) << 4) | (four(w.z) << 8) | (four(w.w) << 12);
}

// DashMap::get(&(position, content_hash)) from slot h on, walked in the tag bytes: the aligned 32 B tag sector holding h is read, the
// chain is followed there up to its first empty tag (the next sector only when the chain runs past this one's end, wrapping at the
// mask), and a 32 B slot is loaded only where the tag equals the key's; its full key is then compared, so a tag collision costs one
// slot read and never a wrong answer.  Per-thread (divergent).  The walk is split in three steps so that a caller with two lookups can
// have both tag loads, then both slot loads in flight together: tag_sector, the load of tag_slot, tag_finish.
__device__ __forceinline__ uint32_t tag_rep(uint32_t pos, uint64_t content) { return (uint32_t)tag_of(pos, content) * 0x01010101u; }
struct TagCursor { uint32_t base, cand; bool ends; };   // one tag sector: the candidate slots left in it, and whether the chain ends in it
__device__ __forceinline__ TagCursor tag_sector(const EventIndexView& v, uint32_t rep, uint32_t h) {
    const uint32_t base = h & ~31u;   // capacity ≥ 1024: a sector never straddles the end of the table
    const uint4 t0 = ld_tags(v.tags + base), t1 = ld_tags(v.tags + base + 16);
    const uint32_t from = ~0u << (h & 31u);
    const uint32_t empty = (byte_eq_bits(t0, 0u) | (byte_eq_bits(t1, 0u) << 16)) & from;
    uint32_t cand = (byte_eq_bits(t0, rep) | (byte_eq_bits(t1, rep) << 16)) & from;
    if (empty) cand &= (empty & (0u - empty)) - 1u;   // only the slots before the first empty one
    return TagCursor{base, cand, empty != 0};
}
__device__ __forceinline__ uint32_t tag_slot(const TagCursor& c) { return c.base + (uint32_t)(__ffs((int)c.cand) - 1); }
__device__ __forceinline__ bool key_is(const Slot& s, uint32_t pos, uint64_t content) {
    return s.state != SLOT_EMPTY && s.state != SLOT_TOMB && s.content == content && s.pos == pos;
}
// `s` is slot tag_slot(c) when c.cand is non-zero (loaded by the caller)
__device__ __forceinline__ bool tag_finish(const EventIndexView& v, uint32_t pos, uint64_t content, uint32_t rep, TagCursor c, Slot s, Slot& out) {
#pragma unroll 1
    for (;;) {
        while (c.cand) {
            if (key_is(s, pos, content)) { out = s; return true; }
            c.cand &= c.cand - 1u;
            if (c.cand) s = load_slot(v.slots + tag_slot(c));
        }
        if (c.ends) return false;
        c = tag_sector(v, rep, (c.base + 32u) & v.mask);
        if (c.cand) s = load_slot(v.slots + tag_slot(c));
    }
}
__device__ __forceinline__ bool tag_walk(const EventIndexView& v, uint32_t pos, uint64_t content, uint32_t h, Slot& out) {
    const uint32_t rep = tag_rep(pos, content);
    const TagCursor c = tag_sector(v, rep, h);
    Slot s{0, 0, SLOT_EMPTY, 0, 0};
    if (c.cand) s = load_slot(v.slots + tag_slot(c));
    return tag_finish(v, pos, content, rep, c, s, out);
}
// The same lookup from the key's home slot: no slot is read for an absent key unless its tag collides.
__device__ __forceinline__ bool tag_probe(const EventIndexView& v, uint32_t pos, uint64_t content, Slot& out) {
    return tag_walk(v, pos, content, slot_hash(pos, content) & v.mask, out);
}
// The rest of a lookup whose home slot h has been read into s: done when s is empty or is the key, else the chain goes on in the tags.
__device__ __forceinline__ bool finish_probe(const EventIndexView& v, uint32_t pos, uint64_t content, uint32_t h, Slot& s) {
    if (s.state == SLOT_EMPTY) return false;
    if (s.state != SLOT_TOMB && s.content == content && s.pos == pos) return true;
    if (tag_walk(v, pos, content, (h + 1) & v.mask, s)) return true;
    s.state = SLOT_EMPTY;   // as a walk over the slots would have left it: the empty slot that ended the chain
    return false;
}

// DashMap::get(&(position, content_hash)) — the home slot first (hot entries are L2 hits), the collision chain in the tags.  Works
// per-thread (divergent) or warp-uniform (same address in every lane → one broadcast transaction).
__device__ __forceinline__ bool probe(const EventIndexView& v, uint32_t pos, uint64_t content, Slot& out) {
    const uint32_t h = slot_hash(pos, content) & v.mask;
    Slot s = load_slot(v.slots + h);
    if (!finish_probe(v, pos, content, h, s)) return false;
    out = s;
    return true;
}

// ---- worker sets --------------------------------------------------------------------------------------------
template <bool W1> __device__ __forceinline__ uint64_t load_set(const EventIndexView& v, uint64_t payload, int lane) {
    if (W1) return payload;
    return (uint32_t)lane < v.words ? __ldg(v.rows + (size_t)(uint32_t)payload * v.words + lane) : 0ULL;
}
template <bool W1> __device__ __forceinline__ uint32_t set_popc(uint64_t s) {
    if (W1) return (uint32_t)__popcll(s);
    return __reduce_add_sync(FULL, (uint32_t)__popcll(s));
}
template <bool W1> __device__ __forceinline__ bool set_any(uint64_t s) {
    if (W1) return s != 0;
    return __any_sync(FULL, s != 0);
}
// popcount of a whole set by ONE lane (scan path: every lane sizes the entry it probed itself)
template <bool W1> __device__ __forceinline__ uint32_t lane_popc_set(const EventIndexView& v, uint64_t payload) {
    if (W1) return (uint32_t)__popcll(payload);
    const uint64_t* r = v.rows + (size_t)(uint32_t)payload * v.words;
    uint32_t c = 0;
    for (uint32_t i = 0; i < v.words; ++i) c += (uint32_t)__popcll(__ldg(r + i));
    return c;
}

// rolling prefix hash, computed lazily and only when a Multi entry needs it (event_tree.rs:486-501)
struct PrefixCache { int pos; uint64_t val; };
__device__ __forceinline__ uint64_t prefix_at(const uint64_t* ch, int p, PrefixCache& pc) {
    if (pc.pos < 0 || p < pc.pos) { pc.pos = 0; pc.val = ch[0]; }
    while (pc.pos < p) { ++pc.pos; pc.val = xxh3_pair(pc.val, ch[pc.pos], kSeed); }
    return pc.val;
}

// workers_if_single() / SeqEntry::get(prefix) (event_tree.rs:216-235); warp-uniform slot
template <bool W1>
__device__ __forceinline__ bool entry_set(const EventIndexView& v, uint32_t state, uint64_t payload, const uint64_t* ch, int p, int lane,
                                          PrefixCache& pc, uint64_t& set) {
    if (state == SLOT_SINGLE) { set = load_set<W1>(v, payload, lane); return true; }
    uint64_t want = prefix_at(ch, p, pc);
    for (uint32_t i = (uint32_t)payload; i != kNil;) {
        MultiNode nd = load_node(v.multi + i);
        if (nd.prefix == want) { set = load_set<W1>(v, nd.payload, lane); return true; }
        i = nd.next;
    }
    return false;
}

// ---- event sinks: what happens when workers leave the active set at `pos` (score = pos) -------------------
template <bool W1> struct SelectSink {  // keeps only what the argmax can still need
    uint64_t elig, last;
    uint32_t last_score;
    __device__ __forceinline__ void on_event(uint32_t pos, uint64_t set) {
        uint64_t e = set & elig;
        if (set_any<W1>(e)) { last = e; last_score = pos; }
    }
};
template <bool W1> struct DumpSink {  // OverlapScores.scores materialised (find_matches API)
    uint32_t* scores;
    int lane;
    __device__ __forceinline__ void on_event(uint32_t pos, uint64_t set) {
        if (W1) {
            if ((set >> lane) & 1) scores[lane] = pos;
            if ((set >> (lane + 32)) & 1) scores[lane + 32] = pos;
        } else {
            uint64_t w = set;
            while (w) { int b = __ffsll((long long)w) - 1; w &= w - 1; scores[lane * 64 + b] = pos; }
        }
    }
};

// linear_scan_drain (event_tree.rs:582-657) over positions lo..=hi.  All positions of a 32-wide chunk are probed
// in parallel (one lane each); positions that provably leave `active` untouched (Single entry whose set is at
// least as large as the active set — the reference's retain guard) are skipped by ballot, the rest are resolved
// in order.
template <bool W1, class Sink>
__device__ __forceinline__ void scan_drain(const EventIndexView& v, const uint64_t* ch, int lo, int hi, int lane, uint64_t& active,
                                           Sink& sink, PrefixCache& pc) {
    for (int base = lo; base <= hi; base += 32) {
        if (!set_any<W1>(active)) break;
        int p = base + lane;
        bool in_range = p <= hi;
        Slot my{0, 0, SLOT_EMPTY, 0, 0};
        bool found = false;
        uint32_t cnt = 0;
        if (in_range) {
            found = probe(v, (uint32_t)p, ch[p], my);
            if (found && my.state == SLOT_SINGLE) cnt = lane_popc_set<W1>(v, my.payload);
        }
        unsigned remaining = __ballot_sync(FULL, in_range);
        while (remaining) {
            if (!set_any<W1>(active)) break;
            uint32_t nact = set_popc<W1>(active);
            bool noop = found && my.state == SLOT_SINGLE && cnt >= nact;
            unsigned b = __ballot_sync(FULL, in_range && !noop) & remaining;
            if (!b) break;
            int k = __ffs((int)b) - 1;
            int kp = base + k;
            bool kfound = __shfl_sync(FULL, (int)found, k) != 0;
            if (!kfound) { sink.on_event((uint32_t)kp, active); active = 0; break; }
            uint32_t kstate = __shfl_sync(FULL, my.state, k);
            uint64_t kpayload = shfl64(my.payload, k);
            uint64_t ws;
            if (!entry_set<W1>(v, kstate, kpayload, ch, kp, lane, pc, ws)) { sink.on_event((uint32_t)kp, active); active = 0; break; }
            if (set_popc<W1>(ws) < nact) {
                uint64_t drained = active & ~ws;
                sink.on_event((uint32_t)kp, drained);
                active &= ws;
            }
            remaining &= ~((2u << k) - 1u);
        }
    }
}

// jump_search_matches (event_tree.rs:659-753).  `ch[0..len)` content hashes (shared memory), len ≥ 1.
// On return the survivors (score = len) are returned; drained workers were reported through the sink.
//
// The jump destinations 0, J, 2J, …, len-1 do not depend on the data (current_pos always advances to next_pos,
// :721/:733), so they are probed SPECULATIVELY in parallel — one lane per destination, 32 at a time — and the
// count-only jump test (:720) is then replayed in order from registers.  Only a failed test costs a second
// memory round trip (scan_drain).  For len ≤ J+1 (BASELINE config 2: 32 blocks, jump 64) that is exactly the
// reference's two probes, issued concurrently.
template <bool W1, class Sink>
__device__ __forceinline__ uint64_t jump_search(const EventIndexView& v, const uint64_t* ch, int len, int lane, Sink& sink, bool early_exit) {
    PrefixCache pc{-1, 0};
    const uint64_t J = v.jump;
    const int last = len - 1;
    const int m = last == 0 ? 0 : (int)(((uint64_t)last + J - 1) / J);  // destinations after position 0
    uint64_t active = 0;
    int cur = 0;
    for (int base = 0; base <= m; base += 32) {
        const int di = base + lane;
        const bool in_range = di <= m;
        int dpos = 0;
        if (in_range) { uint64_t q = (uint64_t)di * J; dpos = q < (uint64_t)last ? (int)q : last; }
        Slot my{0, 0, SLOT_EMPTY, 0, 0};
        bool found = false;
        uint32_t cnt = 0;
        if (in_range) {
            found = probe(v, (uint32_t)dpos, ch[dpos], my);
            if (!W1 && found && my.state == SLOT_SINGLE) cnt = lane_popc_set<W1>(v, my.payload);
        }
        const int nloc = (m - base + 1) < 32 ? (m - base + 1) : 32;
        for (int k = 0; k < nloc; ++k) {
            const int kd = base + k;
            int kpos;
            { uint64_t q = (uint64_t)kd * J; kpos = q < (uint64_t)last ? (int)q : last; }
            const bool kfound = __shfl_sync(FULL, (int)found, k) != 0;
            const uint32_t kstate = __shfl_sync(FULL, my.state, k);
            const uint64_t kpayload = shfl64(my.payload, k);
            if (kd == 0) {
                if (!kfound) return 0;
                if (!entry_set<W1>(v, kstate, kpayload, ch, 0, lane, pc, active)) return 0;
                if (!set_any<W1>(active)) return 0;
                if (early_exit) { sink.on_event(1, active); return 0; }
                continue;
            }
            uint32_t count = 0;  // count_workers_at(kpos) (:555-574)
            if (kfound) {
                if (kstate == SLOT_SINGLE) count = W1 ? (uint32_t)__popcll(kpayload) : __shfl_sync(FULL, cnt, k);
                else { uint64_t ws; if (entry_set<W1>(v, kstate, kpayload, ch, kpos, lane, pc, ws)) count = set_popc<W1>(ws); }
            }
            if (count != set_popc<W1>(active)) scan_drain<W1>(v, ch, cur + 1, kpos, lane, active, sink, pc);
            cur = kpos;
            if (!set_any<W1>(active)) return 0;
        }
    }
    return active;
}

// ---- K2b part 1: content hashes — a pure streaming kernel ----------------------------------------------------
// One THREAD per block of tokens (64 B at block_size 16: 4×LDG.128, consecutive threads → consecutive blocks, a warp
// streams 2 KB).  Hashes land in a scratch laid out [request][max_blocks] that the search kernel reads back from L2.
// HBM-bound by construction: 4·T bytes in, 8·P bytes out per request, ~110 integer instructions per 64 B.
// tokens are read once: evict-first in L2 (L1 as usual — a thread's four 16 B loads share sectors), so that the stream does not push the
// index slots the same kernel prefetches (evict-last) for the search out of L2 before the search gets to them.  ld.global.cs (evict-first
// in L1 too) was measured slower, most of all in steady state — the second half of every sector came from L2 again.
__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    uint4 r;
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
// the 16 tokens of one block: four evict-first 16 B loads when the block is 16 B aligned, scalar loads otherwise
__device__ __forceinline__ void load_block16(const uint32_t* __restrict__ p, uint32_t (&w)[16]) {
    if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
        const uint4* q = reinterpret_cast<const uint4*>(p);
#pragma unroll
        for (int i = 0; i < 4; ++i) { uint4 t = ld_stream(q + i); w[4 * i] = t.x; w[4 * i + 1] = t.y; w[4 * i + 2] = t.z; w[4 * i + 3] = t.w; }
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = __ldg(p + i);
    }
}
// two blocks of one request: they lie a multiple of 64 B apart, so one alignment test serves both, and all their loads are issued before
// either block is hashed (two separate load_block16 branches let the compiler hash the first block before loading the second)
__device__ __forceinline__ void load_block16_pair(const uint32_t* __restrict__ p0, const uint32_t* __restrict__ p1, uint32_t (&w0)[16], uint32_t (&w1)[16]) {
    if ((reinterpret_cast<uintptr_t>(p0) & 15) == 0) {
        const uint4* q0 = reinterpret_cast<const uint4*>(p0);
        const uint4* q1 = reinterpret_cast<const uint4*>(p1);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint4 t0 = ld_stream(q0 + i), t1 = ld_stream(q1 + i);
            w0[4 * i] = t0.x; w0[4 * i + 1] = t0.y; w0[4 * i + 2] = t0.z; w0[4 * i + 3] = t0.w;
            w1[4 * i] = t1.x; w1[4 * i + 1] = t1.y; w1[4 * i + 2] = t1.z; w1[4 * i + 3] = t1.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) { w0[i] = __ldg(p0 + i); w1[i] = __ldg(p1 + i); }
    }
}
template <int BS>
__device__ __forceinline__ uint64_t hash_block(const uint32_t* __restrict__ p, uint32_t bs) {
    if (BS == 16) {
        uint32_t w[16];
        load_block16(p, w);
        return xxh3_16words(w, kSeed);
    }
    return xxh3_words(p, bs, kSeed);
}

template <int BS>   // BS = 16: the common block size, fully unrolled; BS = 0: any run-time block size
__global__ void __launch_bounds__(256, 8) hash_blocks_kernel(const __grid_constant__ MultiArgs a) {   // 8 CTAs = 2048 threads per SM: the 64 B per thread in flight are the bandwidth
    // programmatic dependent launch: once every CTA of this grid has started, the search kernel's CTAs may take the slots the last wave frees
    // (they load their fleet tables and then wait for this grid's completion in griddepcontrol.wait); a no-op without a dependent launch
    asm volatile("griddepcontrol.launch_dependents;");
    const BatchDesc& b = a.b[blockIdx.y];
    const uint64_t total = (uint64_t)b.n * a.max_blocks;
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(t / a.max_blocks), blk = (uint32_t)(t % a.max_blocks);
        const uint32_t off = __ldg(b.offsets + r), ntok = __ldg(b.offsets + r + 1) - off;
        const uint32_t bs = BS ? (uint32_t)BS : a.block_size;
        const uint32_t nb = ntok / bs;
        if (blk == 0 && a.recs) a.recs[(uint64_t)b.hash_base + r].ntok = ntok;
        if (blk < nb) {
            const uint64_t h = hash_block<BS>(b.tokens + off + (size_t)blk * bs, bs);
            a.hashes[((uint64_t)b.hash_base + r) * a.max_blocks + blk] = h;
            if (a.recs) {   // the search kernel's phase A reads these instead of walking offsets → hash row
                if (blk == 0) a.recs[(uint64_t)b.hash_base + r].h0 = h;
                if (blk == min(a.pf_jump, nb - 1)) a.recs[(uint64_t)b.hash_base + r].h1 = h;
            }
            // the search kernel probes positions 0 and min(jump, last) first: pull those 32 B slots into L2 now (fire and forget), so that
            // its dependent chain offsets → hashes → slots runs at L2 latency instead of paying a DRAM miss per probe
            if (a.pf_slots && (blk == 0 || blk == min(a.pf_jump, nb - 1)))
                asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(reinterpret_cast<const Slot*>(a.pf_slots) + (slot_hash(blk, h) & a.pf_mask)));
        }
    }
    if (a.ready) {   // concurrent split launch: this CTA's share of batch blockIdx.y is in memory
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) atomicAdd(a.ready + blockIdx.y, 1u);
    }
}

// ---- K3: max_by_key((score, Reverse(load), Reverse(tree_size))) with LAST max = highest slice index ---------
struct Cand {
    bool have; uint64_t ld, ts; int32_t sl;
    __device__ __forceinline__ void consider(int32_t s, uint64_t l, uint64_t t) {
        bool better = !have || l < ld || (l == ld && (t < ts || (t == ts && s > sl)));
        if (better) { have = true; ld = l; ts = t; sl = s; }
    }
};

__device__ __forceinline__ void write_pick(const BatchDesc& b, uint32_t r, int32_t out, uint32_t branch, uint32_t matched, uint32_t ntok) {
    b.out_idx[r] = out;
    if (b.out_info) {
        smgx_decision_info di;
        di.matched = matched; di.input = ntok; di.branch = (uint8_t)branch;
        di.nodes = 0; di.reserved[0] = di.reserved[1] = 0;
        b.out_info[r] = di;
    }
}

// ---- search + pick, fleets of ≤ 64 interned workers: ONE THREAD per request ---------------------------------
// Worker sets are single u64 words held in the slot itself, so the whole jump search is scalar code: two
// independent slot loads up front (position 0 and the first jump destination), the count test, and only on a
// failed test the linear drain (4 probes in flight at a time).  ~30 warp-instructions per request on the common
// path; the kernel is a few microseconds for 10^5 requests and disappears next to the hash stream.
__device__ __forceinline__ bool t_entry_set(const EventIndexView& v, const Slot& s, const uint64_t* ch, int p, PrefixCache& pc, uint64_t& set) {
    if (s.state == SLOT_SINGLE) { set = s.payload; return true; }
    uint64_t want = prefix_at(ch, p, pc);
    for (uint32_t i = (uint32_t)s.payload; i != kNil;) {
        MultiNode nd = load_node(v.multi + i);
        if (nd.prefix == want) { set = nd.payload; return true; }
        i = nd.next;
    }
    return false;
}
// The scalar part of jump_search_matches (event_tree.rs:659-753): everything except linear_scan_drain.  A thread runs
// until it is finished or until a count test fails (:720) — then it parks with the range to drain, and the WARP drains
// it cooperatively (scan_drain<true>: 32 positions probed in parallel) before the thread resumes.
struct ThreadSearch {
    const uint64_t* ch;
    uint64_t active, last;
    uint32_t last_score;
    int len, cur, lo, hi;
    bool done, need;
};

__global__ void __launch_bounds__(128) event_search_thread_kernel(EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a) {
    __shared__ int32_t s_slice[64];
    __shared__ uint64_t s_load[64], s_ts[64];
    if (threadIdx.x < 64) {
        bool ok = threadIdx.x < v.n_workers;
        s_slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        s_load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        s_ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const BatchDesc& b = a.b[blockIdx.y];
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = r < b.n;
    const FleetDerived fd = *f.derived;
    const uint64_t elig = f.elig[0];
    const uint64_t J = v.jump;

    uint32_t ntok = 0, nb = 0, branch = SMGX_BR_NO_HEALTHY;
    int32_t out = -1;
    ThreadSearch st{nullptr, 0, 0, 0, 0, 0, 0, 0, true, false};
    // speculative second probe (first jump destination), consumed by the first count test
    Slot s1{0, 0, SLOT_EMPTY, 0, 0};
    uint64_t c1 = 0;
    uint32_t h1 = 0;
    int next0 = 0;
    bool have1 = false;
    PrefixCache pc{-1, 0};
    bool searching = false;
    const bool cand_mode = b.cand != nullptr;   // sharded fleet: the healthy/imbalance shortcuts are global decisions (reduce step)
    if (valid) {
        const uint32_t off = __ldg(b.offsets + r);
        ntok = __ldg(b.offsets + r + 1) - off;
        if (!cand_mode && fd.n_healthy == 0) {
        } else if (!cand_mode && fd.imbalanced) {
            out = fd.min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD;
        } else {
            nb = a.block_size ? ntok / a.block_size : 0;
            if (nb > a.max_blocks) { atomicExch(a.err_flag, 1u); branch = 255; }
            else {
                branch = SMGX_BR_EVENT_MIN_LOAD;   // until an overlap is found
                if (nb > 0 && v.n_workers > 0) {
                    st.ch = a.hashes + ((uint64_t)b.hash_base + r) * a.max_blocks;
                    st.len = (int)nb;
                    const int last = st.len - 1;
                    next0 = last == 0 ? 0 : ((uint64_t)last > J ? (int)J : last);
                    const uint64_t c0 = st.ch[0];
                    c1 = st.ch[next0];
                    const uint32_t h0 = slot_hash(0, c0) & v.mask;
                    h1 = slot_hash((uint32_t)next0, c1) & v.mask;
                    Slot s0 = load_slot(v.slots + h0);
                    s1 = load_slot(v.slots + h1);          // both probes in flight together
                    have1 = last > 0;
                    if (finish_probe(v, 0, c0, h0, s0) && t_entry_set(v, s0, st.ch, 0, pc, st.active) && st.active) {
                        st.done = false;
                        searching = true;
                    }
                }
            }
        }
    }
    for (;;) {
        if (!st.done && !st.need) {
            const int last = st.len - 1;
            while (st.cur < last && st.active) {
                const int next = ((uint64_t)(last - st.cur) > J) ? st.cur + (int)J : last;
                Slot s;
                bool fnd;
                if (have1 && next == next0) { fnd = finish_probe(v, (uint32_t)next, c1, h1, s1); s = s1; have1 = false; }
                else fnd = probe(v, (uint32_t)next, st.ch[next], s);
                uint32_t count = 0;
                uint64_t ws;
                if (fnd && t_entry_set(v, s, st.ch, next, pc, ws)) count = (uint32_t)__popcll(ws);
                if (count != (uint32_t)__popcll(st.active)) { st.need = true; st.lo = st.cur + 1; st.hi = next; break; }
                st.cur = next;
            }
            if (!st.need) st.done = true;
        }
        unsigned m = __ballot_sync(FULL, st.need);
        if (!m) {
            if (__all_sync(FULL, st.done)) break;
            continue;
        }
        while (m) {
            const int L = __ffs((int)m) - 1;
            m &= m - 1;
            const uint64_t* lch = reinterpret_cast<const uint64_t*>(shfl64(reinterpret_cast<uint64_t>(st.ch), L));
            const int llo = __shfl_sync(FULL, st.lo, L), lhi = __shfl_sync(FULL, st.hi, L);
            uint64_t lact = shfl64(st.active, L);
            SelectSink<true> sk{elig, 0, 0};
            PrefixCache wpc{-1, 0};
            scan_drain<true>(v, lch, llo, lhi, lane, lact, sk, wpc);
            if (lane == L) {
                st.active = lact;
                if (sk.last) { st.last = sk.last; st.last_score = sk.last_score; }
                st.need = false;
                st.cur = st.hi;
            }
        }
    }
    if (!valid) return;
    uint32_t matched = 0;
    Cand c{false, 0, 0, -1};
    if (searching) {
        uint64_t winset = st.active & elig;
        uint32_t score = nb;
        if (!winset) { winset = st.last; score = st.last_score; }
        if (winset) {
            uint64_t w = winset;
            while (w) { int id = __ffsll((long long)w) - 1; w &= w - 1; c.consider(s_slice[id], s_load[id], s_ts[id]); }
            out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = score;
        }
    }
    if (cand_mode) {
        smgx_shard_candidate sc;
        sc.score = c.have ? matched : 0; sc.local_idx = c.have ? (uint32_t)c.sl : 0xFFFFFFFFu; sc.load = c.ld; sc.tree_size = c.ts;
        b.cand[r] = sc;
        return;
    }
    if (branch == SMGX_BR_EVENT_MIN_LOAD) out = fd.min_load_idx;
    write_pick(b, r, out, branch, matched, ntok);
}

// ---- search + pick, wider fleets (65..2048 interned workers): one WARP per request, one u64 set word per lane ----
__device__ __forceinline__ Cand warp_arg_best(const EventIndexView& v, const FleetView& f, uint64_t winset, int lane) {
    Cand c{false, 0, 0, -1};
    uint64_t w = winset;
    while (w) {
        int bit = __ffsll((long long)w) - 1;
        w &= w - 1;
        uint32_t id = (uint32_t)(lane * 64 + bit);
        c.consider(f.slice_of_id[id], f.load_of_id[id], v.tree_sizes[id]);
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
        bool oh = __shfl_xor_sync(FULL, (int)c.have, d) != 0;
        uint64_t ol = shfl64_xor(c.ld, d), ot = shfl64_xor(c.ts, d);
        int32_t os = __shfl_xor_sync(FULL, c.sl, d);
        if (oh) c.consider(os, ol, ot);
    }
    return c;
}

__global__ void __launch_bounds__(256) event_search_warp_kernel(EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a) {
    extern __shared__ uint64_t smem_ch[];
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    uint64_t* ch = smem_ch + (size_t)wic * a.max_blocks;
    const FleetDerived fd = *f.derived;
    const uint64_t elig = (uint32_t)lane < v.words ? f.elig[lane] : 0ULL;
    const BatchDesc& b = a.b[blockIdx.y];
    const bool cand_mode = b.cand != nullptr;
    for (uint32_t r = blockIdx.x * wpc + wic; r < b.n; r += gridDim.x * wpc) {
        const uint32_t off = b.offsets[r], ntok = b.offsets[r + 1] - off;
        int32_t out = -1;
        uint32_t branch = SMGX_BR_NO_HEALTHY, matched = 0;
        Cand best{false, 0, 0, -1};
        if (!cand_mode && fd.n_healthy == 0) {
        } else if (!cand_mode && fd.imbalanced) {
            out = fd.min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD;
        } else {
            const uint32_t nb = a.block_size ? ntok / a.block_size : 0;
            if (nb > a.max_blocks) { if (lane == 0) atomicExch(a.err_flag, 1u); branch = 255; }
            else {
                uint64_t winset = 0;
                uint32_t score = 0;
                if (nb > 0 && v.n_workers > 0) {
                    const uint64_t* gh = a.hashes + ((uint64_t)b.hash_base + r) * a.max_blocks;
                    for (uint32_t i = lane; i < nb; i += 32) ch[i] = gh[i];
                    __syncwarp();
                    SelectSink<false> sink{elig, 0, 0};
                    uint64_t surv = jump_search<false>(v, ch, (int)nb, lane, sink, false) & elig;
                    if (set_any<false>(surv)) { winset = surv; score = nb; }
                    else { winset = sink.last; score = sink.last_score; }
                    __syncwarp();
                }
                if (set_any<false>(winset)) { best = warp_arg_best(v, f, winset, lane); out = best.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = score; }
                else { out = fd.min_load_idx; branch = SMGX_BR_EVENT_MIN_LOAD; }
            }
        }
        if (cand_mode) {
            if (lane == 0) {
                smgx_shard_candidate sc;
                sc.score = best.have ? matched : 0; sc.local_idx = best.have ? (uint32_t)best.sl : 0xFFFFFFFFu; sc.load = best.ld; sc.tree_size = best.ts;
                b.cand[r] = sc;
            }
            continue;
        }
        if (lane == 0) write_pick(b, r, out, branch, matched, ntok);
    }
}

// ---- the whole event-driven pick in ONE kernel: hash → search → pick, one warp per request, software-pipelined --------------
// The split design above needs two launches and a 256 B/request hash scratch, and its search kernel is a partial wave of dependent
// loads that only disappears when other launches overlap it.  Here a persistent warp walks requests g, g+S, g+2S, …; while it hashes
// and probes for request g, the 2 KB token load of request g+S (one 64 B block per lane, 4×LDG.128) and the offsets of request g+2S
// are already in flight — the token stream never pauses for the probe latency, every token is read exactly once, the hashes never
// leave the SM, and a launch of K batches is one grid.
//   ← compute_request_content_hashes + PositionalIndexer::find_matches + score_overlap   event_tree.rs:141-151, :461-753; cache_aware.rs:736-831
//
// The kernel is co-limited by instruction issue (ncu, first version), so the
// common shapes take a FAST PATH that never leaves registers: a request of ≤ 32 blocks whose jump search is one jump (jump_size ≥
// blocks − 1: BASELINE config 2) probes positions 0 and last from the two lanes that hold those hashes, and decides from two shuffled
// slots: miss at 0 → no overlap; Single at 0 and a Single at `last` of equal cardinality (the reference's count-only jump test, :720)
// → the position-0 set survives with score = blocks.  Everything else (a failed count test → linear drain, Multi entries, longer
// requests, more than one jump, fleets above 64 workers) goes through the generic warp-cooperative jump_search on a per-warp
// shared-memory row of hashes — a __noinline__ call, so its registers do not tax the fast path.
struct FusedPos { uint32_t j, r; };   // batch index, request index inside the batch

__device__ __forceinline__ void fused_advance(const MultiArgs& a, FusedPos& p, uint32_t by) {
    p.r += by;
    while (p.j < a.count && p.r >= a.b[p.j].n) { p.r -= a.b[p.j].n; ++p.j; }
}
struct SlowResult { uint64_t winset; uint32_t score; };
// generic search on the shared-memory hash row; returns the eligible set the argmax runs over (survivors, else the latest eligible drained set)
template <bool W1>
__device__ __forceinline__ SlowResult slow_search_inline(const EventIndexView& v, const uint64_t* ch, int nb, int lane, uint64_t elig) {
    SelectSink<W1> sink{elig, 0, 0};
    const uint64_t surv = jump_search<W1>(v, ch, nb, lane, sink, false) & elig;
    SlowResult r;
    if (set_any<W1>(surv)) { r.winset = surv; r.score = (uint32_t)nb; }
    else { r.winset = sink.last; r.score = sink.last_score; }
    return r;
}
template <bool W1>
__device__ __noinline__ SlowResult fused_slow_search(const EventIndexView* vp, const uint64_t* ch, int nb, int lane, uint64_t elig) {
    const EventIndexView v = *vp;
    SelectSink<W1> sink{elig, 0, 0};
    const uint64_t surv = jump_search<W1>(v, ch, nb, lane, sink, false) & elig;
    SlowResult r;
    if (set_any<W1>(surv)) { r.winset = surv; r.score = (uint32_t)nb; }
    else { r.winset = sink.last; r.score = sink.last_score; }
    return r;
}

// argmax + store for one request (any single thread): `win` = eligible workers tied on the best overlap `score` (0: the least-loaded
// healthy worker); a worker-id-sharded fleet stores this shard's candidate instead of a pick
__device__ __forceinline__ void finish_pick(const BatchDesc& b, uint32_t r, const int32_t* s_slice, const uint64_t* s_load, const uint64_t* s_ts,
                                            int32_t min_load_idx, uint64_t win, uint32_t score, uint32_t ntok) {
    int32_t out = min_load_idx;
    uint32_t branch = SMGX_BR_EVENT_MIN_LOAD, matched = 0;
    Cand c{false, 0, 0, -1};
    if (win) {
        while (win) { int id = __ffsll((long long)win) - 1; win &= win - 1; c.consider(s_slice[id], s_load[id], s_ts[id]); }
        out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = score;
    }
    if (b.cand) {
        smgx_shard_candidate sc;
        sc.score = c.have ? matched : 0; sc.local_idx = c.have ? (uint32_t)c.sl : 0xFFFFFFFFu; sc.load = c.ld; sc.tree_size = c.ts;
        b.cand[r] = sc;
    } else write_pick(b, r, out, branch, matched, ntok);
}

// linear_scan_drain over positions 1..=last (event_tree.rs:582-657) of a request of nb ≤ 32 blocks whose count test failed, from registers:
// lane p ≤ last holds its probe of position p (found, sl), lane 0's being the Single entry the jump search started from.  The reference's
// ordered scan with its retain guard is replayed by a ballot loop.  Warp-uniform result: the tied set and its score, or bail = an entry
// that needs the rolling prefix hash (Multi) was met, and the generic search has to decide.
struct DrainResult { uint64_t win; uint32_t score; bool bail; };
__device__ __forceinline__ DrainResult drain_resolve(int nb, uint64_t elig, int lane, bool found, const Slot& sl) {
    const int last = nb - 1;
    uint64_t active = shfl64(sl.payload, 0);
    const bool in_range = lane >= 1 && lane <= last;
    const uint32_t cnt = (found && sl.state == SLOT_SINGLE) ? (uint32_t)__popcll(sl.payload) : 0;
    uint64_t last_set = 0;
    uint32_t last_score = 0;
    bool bail = !__shfl_sync(FULL, (int)found, 0) || __shfl_sync(FULL, sl.state, 0) != SLOT_SINGLE;
    unsigned remaining = __ballot_sync(FULL, in_range);
    while (!bail && remaining && active) {
        const uint32_t nact = (uint32_t)__popcll(active);
        const bool noop = found && sl.state == SLOT_SINGLE && cnt >= nact;           // retain guard (:611, :641)
        const unsigned bm = __ballot_sync(FULL, in_range && !noop) & remaining;
        if (!bm) break;
        const int k = __ffs((int)bm) - 1;
        if (!__shfl_sync(FULL, (int)found, k)) {                                     // missing entry drains everything (:598-604)
            const uint64_t e = active & elig;
            if (e) { last_set = e; last_score = (uint32_t)k; }
            active = 0;
            break;
        }
        if (__shfl_sync(FULL, sl.state, k) != SLOT_SINGLE) { bail = true; break; }
        const uint64_t ws = shfl64(sl.payload, k);
        if ((uint32_t)__popcll(ws) < nact) {
            const uint64_t e = active & ~ws & elig;
            if (e) { last_set = e; last_score = (uint32_t)k; }
            active &= ws;
        }
        remaining &= ~((2u << k) - 1u);
    }
    DrainResult d{active & elig, (uint32_t)nb, bail};
    if (!d.win) { d.win = last_set; d.score = last_score; }
    return d;
}

// ---- search + pick, fleets of ≤ 64 interned workers, second version: balanced drains -------------------------------------------
// event_search_thread_kernel above is one partial wave whose duration is set by its UNLUCKIEST warp: every request whose count test
// fails (a stored prefix shorter than the request: ≈ 10 % of BASELINE config 2) is drained in its home warp, one after another, two to
// three dependent memory round trips each — the warp that happens to hold nine of them finishes long after the one that holds none
// (the launch time hardly depends on its size; few warps stay active).  Here a CTA of 256 requests runs three phases:
//   A  one THREAD per request: offsets, the two jump-destination hashes from the scratch, both probes in flight together, the count-only
//      jump test (event_tree.rs:720).  Done for full hits and novel requests; otherwise the request is pushed onto a shared-memory queue;
//   B  the queue is spread over the CTA's 8 warps (≈ 3 drains per warp instead of up to ≈ 10): lane p loads hash p (one coalesced 256 B
//      read), every position 1..last is probed at once, the reference's ordered scan with its retain guard is replayed from registers by
//      a ballot loop — ONE round trip per drain;
//   C  whatever needs rolling prefix hashes or more than one jump (Multi entries, > 32 blocks, jump_size < blocks − 1) runs the generic
//      warp-cooperative jump_search on a shared-memory row, again spread over the warps.
struct Search2Item { uint32_t r; uint32_t nb; };

struct Search2Smem {
    int32_t slice[64];
    uint64_t load[64], ts[64];
    Search2Item qb[256], qc[256];
    uint32_t nb, nc, last;
};
// The three phases for r_count ≤ 256 requests of batch `by` starting at r_begin, run by a whole CTA of 256 threads.  WAIT: the stand-alone search
// kernel launched beside the hash kernel (a.ready).  CG: records and hash rows were written by OTHER CTAs of the running kernel
// (event_hs_kernel) — read them from L2 (ld.global.cg), never through this SM's L1.
template <int NT> __device__ __forceinline__ void search2_sync() {   // the NT threads running search2_body (NT < 256: named barrier 1)
    if (NT == 256) __syncthreads();
    else asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
}
template <bool WAIT, bool CG, int NT = 256>
__device__ __forceinline__ void search2_body(const EventIndexView& v, const FleetView& f, const MultiArgs& a, const uint32_t by, const uint32_t r_begin,
                                             const uint32_t r_count, Search2Smem& sm, uint64_t* smem_ch, const uint32_t tile_req = 256,
                                             const uint32_t tile_stride = 0) {
    int32_t (&s_slice)[64] = sm.slice;
    uint64_t (&s_load)[64] = sm.load;
    uint64_t (&s_ts)[64] = sm.ts;
    Search2Item (&s_qb)[256] = sm.qb;
    Search2Item (&s_qc)[256] = sm.qc;
    uint32_t& s_nb = sm.nb;
    uint32_t& s_nc = sm.nc;
    auto ld_rec = [&](uint64_t i) -> SearchRec {
        if (!CG) return a.recs[i];
        const uint4* q = reinterpret_cast<const uint4*>(a.recs + i);
        const uint4 lo = __ldcg(q), hi = __ldcg(q + 1);
        SearchRec rr;
        rr.h0 = (uint64_t)lo.x | ((uint64_t)lo.y << 32); rr.h1 = (uint64_t)lo.z | ((uint64_t)lo.w << 32);
        rr.ntok = hi.x;
        return rr;
    };
    auto ld_hash = [&](const uint64_t* p) -> uint64_t { return CG ? (uint64_t)__ldcg(reinterpret_cast<const unsigned long long*>(p)) : *p; };
    if (threadIdx.x < 64) {
        bool ok = threadIdx.x < v.n_workers;
        s_slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        s_load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        s_ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    if (WAIT) asm volatile("griddepcontrol.wait;" ::: "memory");   // launched as a programmatic dependent of the hash kernel: its rows and records are complete and visible from here on
    if (threadIdx.x == 0) {
        s_nb = 0; s_nc = 0;
        if (WAIT && a.ready) {   // launched alongside the hash kernel: wait until every hash CTA of this batch has counted itself in
            const long long t0 = clock64();
            for (;;) {
                uint32_t cur;
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(a.ready + by) : "memory");
                if ((int32_t)(cur - a.ready_target[by]) >= 0) break;
                if (clock64() - t0 > 4000000000LL) { atomicExch(a.err_flag, 3u); break; }   // ≈ 2 s: the hash kernel never ran — report, do not hang
                __nanosleep(100);
            }
        }
    }
    search2_sync<NT>();
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
    const BatchDesc& b = a.b[by];
    const bool cand_mode = b.cand != nullptr;
    const FleetDerived fd = *f.derived;
    const uint64_t elig = f.elig[0];
    auto finish = [&](uint32_t r, uint64_t win, uint32_t score, uint32_t ntok) {
        finish_pick(b, r, s_slice, s_load, s_ts, fd.min_load_idx, win, score, ntok);
    };

    // ---- phase A ----
    // thread t ↔ request t of the range; a range may be a run of equally spaced tiles (event_stream_kernel): tile t / tile_req, slot t % tile_req
    const uint32_t r = r_begin + (threadIdx.x / tile_req) * tile_stride + threadIdx.x % tile_req;
    if (threadIdx.x < r_count) {
        const SearchRec rec = ld_rec((uint64_t)b.hash_base + r);   // one 32 B record written by the hash kernel
        const uint32_t ntok = rec.ntok;
        if (!cand_mode && fd.n_healthy == 0) write_pick(b, r, -1, SMGX_BR_NO_HEALTHY, 0, ntok);
        else if (!cand_mode && fd.imbalanced) write_pick(b, r, fd.min_load_idx, SMGX_BR_IMBALANCED_MIN_LOAD, 0, ntok);
        else {
            const uint32_t nb = a.block_size ? ntok / a.block_size : 0;
            if (nb > a.max_blocks) { atomicExch(a.err_flag, 1u); if (!cand_mode) write_pick(b, r, -1, 255, 0, ntok); else finish(r, 0, 0, ntok); }
            else if (nb == 0 || v.n_workers == 0) finish(r, 0, 0, ntok);
            else if (nb > 32 || nb - 1 > v.jump) { const uint32_t q = atomicAdd(&s_nc, 1u); s_qc[q] = Search2Item{r, nb}; }
            else {
                const int last = (int)nb - 1;
                const uint64_t c0 = rec.h0, c1 = rec.h1;
                const uint32_t h0 = slot_hash(0, c0) & v.mask, h1 = slot_hash((uint32_t)last, c1) & v.mask;
                Slot s0 = load_slot(v.slots + h0), s1 = load_slot(v.slots + h1);          // both probes in flight together (L2-warm: prefetched by the hash kernel)
                if (!finish_probe(v, 0, c0, h0, s0)) finish(r, 0, 0, ntok);               // nothing cached at position 0 (:676-683)
                else if (s0.state != SLOT_SINGLE) { const uint32_t q = atomicAdd(&s_nc, 1u); s_qc[q] = Search2Item{r, nb}; }
                else if (s0.payload == 0 || last == 0) finish(r, s0.payload & elig, nb, ntok);
                else {
                    const bool f1 = finish_probe(v, (uint32_t)last, c1, h1, s1);
                    if (f1 && s1.state != SLOT_SINGLE) { const uint32_t q = atomicAdd(&s_nc, 1u); s_qc[q] = Search2Item{r, nb}; }
                    else if (f1 && __popcll(s1.payload) == __popcll(s0.payload)) finish(r, s0.payload & elig, nb, ntok);   // count-only jump test (:720)
                    else { const uint32_t q = atomicAdd(&s_nb, 1u); s_qb[q] = Search2Item{r, nb}; }
                }
            }
        }
    }
    search2_sync<NT>();

    // ---- phase B: register drains, one warp per queued request, the queue striped over the warps; two requests per round so that the
    //      hash loads and the probes of the second overlap those of the first ----
    const uint32_t n_b = s_nb;
    auto resolve = [&](const Search2Item it, bool found, const Slot& sl) {
        const DrainResult d = drain_resolve((int)it.nb, elig, lane, found, sl);
        if (lane != 0) return;
        if (d.bail) { const uint32_t qq = atomicAdd(&s_nc, 1u); s_qc[qq] = it; }
        else finish(it.r, d.win, d.score, b.out_info ? ld_rec((uint64_t)b.hash_base + it.r).ntok : 0u);   // ntok only feeds out_info: no round trip without it
    };
    constexpr uint32_t NW = NT / 32;
    for (uint32_t q = wic; q < n_b; q += 2 * NW) {
        const Search2Item it0 = s_qb[q];
        const bool two = q + NW < n_b;
        const Search2Item it1 = two ? s_qb[q + NW] : Search2Item{0, 0};
        const uint64_t* ch0 = a.hashes + ((uint64_t)b.hash_base + it0.r) * a.max_blocks;
        const uint64_t* ch1 = a.hashes + ((uint64_t)b.hash_base + it1.r) * a.max_blocks;
        const uint64_t h0 = (uint32_t)lane < it0.nb ? ld_hash(ch0 + lane) : 0;
        const uint64_t h1 = (uint32_t)lane < it1.nb ? ld_hash(ch1 + lane) : 0;
        // every position of both requests probed at once (position 0 again: L2-hot)
        const uint32_t i0 = slot_hash((uint32_t)lane, h0) & v.mask, i1 = slot_hash((uint32_t)lane, h1) & v.mask;
        Slot sl0{0, 0, SLOT_EMPTY, 0, 0}, sl1{0, 0, SLOT_EMPTY, 0, 0};
        if ((uint32_t)lane < it0.nb) sl0 = load_slot(v.slots + i0);
        if ((uint32_t)lane < it1.nb) sl1 = load_slot(v.slots + i1);
        bool f0 = false, f1 = false;
        if ((uint32_t)lane < it0.nb) f0 = finish_probe(v, (uint32_t)lane, h0, i0, sl0);
        if ((uint32_t)lane < it1.nb) f1 = finish_probe(v, (uint32_t)lane, h1, i1, sl1);
        resolve(it0, f0, sl0);
        if (two) resolve(it1, f1, sl1);
    }
    search2_sync<NT>();

    // ---- phase C: generic search ----
    const uint32_t n_c = s_nc;
    uint64_t* row = smem_ch + (size_t)wic * a.max_blocks;
    for (uint32_t q = wic; q < n_c; q += NW) {
        const Search2Item it = s_qc[q];
        const uint64_t* ch = a.hashes + ((uint64_t)b.hash_base + it.r) * a.max_blocks;
        for (uint32_t i = lane; i < it.nb; i += 32) row[i] = ld_hash(ch + i);
        __syncwarp();
        const SlowResult sr = NT == 256 ? fused_slow_search<true>(&v, row, (int)it.nb, lane, elig) : slow_search_inline<true>(v, row, (int)it.nb, lane, elig);
        if (lane == 0) finish(it.r, sr.winset, sr.score, b.out_info ? ld_rec((uint64_t)b.hash_base + it.r).ntok : 0u);
        __syncwarp();
    }
}

template <int RPC>   // requests per CTA handled by phase A (256 threads either way: the queues of phases B / C are spread over all 8 warps)
__global__ void __launch_bounds__(256) event_search2_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a) {
    extern __shared__ uint64_t smem_ch[];                 // [8 warps][max_blocks] for phase C
    __shared__ Search2Smem sm;
    const uint32_t r_begin = blockIdx.x * RPC, n = a.b[blockIdx.y].n;
    search2_body<true, false>(v, f, a, blockIdx.y, r_begin, r_begin < n ? min((uint32_t)RPC, n - r_begin) : 0u, sm, smem_ch);
}

// ---- ONE launch: the hash stream, and the search of every 256-request group run by the LAST hash CTA of that group ------------------
// The pair above costs a lone call a latency tail beyond its streaming time: the search kernel cannot start before the last hash CTA has
// retired, and is itself a chain of dependent round trips.  Here the dependency is resolved per GROUP of 256
// requests instead of per launch.  The grid is the hash kernel's (one thread per UNR slots of the [n][max_blocks] block grid — UNR = 2:
// 128 B in flight per thread, 1024 resident threads per SM hold the same bytes in flight as the stand-alone kernel's 2048 × 64 B, which
// leaves every thread 64 registers, what the search phases need).  A CTA that has stored its hashes and records fences, then counts
// itself into the counter of every group its slots belong to; whoever brings a counter to the group's CTA count is the last writer of
// that group: it resets the counter for the next launch and runs search2_body on the group — one thread per request, all inputs in L2,
// read with ld.global.cg.  Nobody spins, nobody waits: the searches of the early groups run under the hash stream of the later ones,
// and only the last groups' searches (one chain of round trips) remain after the stream ends.
template <int BS, int UNR>
__global__ void __launch_bounds__(256, 4) event_hs_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a) {
    extern __shared__ uint64_t smem_ch[];
    __shared__ Search2Smem sm;
    const BatchDesc& b = a.b[blockIdx.y];
    const uint32_t mb = a.max_blocks;
    const uint64_t total = (uint64_t)b.n * mb;
    const uint64_t t0 = (uint64_t)blockIdx.x * (256u * UNR);
    if (t0 >= total) return;                                  // CTAs beyond this batch's block grid (the grid is sized for the largest batch)
    const uint32_t bs = BS ? (uint32_t)BS : a.block_size;
    {
        uint32_t rr[UNR], blk[UNR], off[UNR], ntok[UNR];
        bool live[UNR];
        uint32_t w[UNR][16];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const uint64_t t = t0 + (uint64_t)u * 256 + threadIdx.x;
            live[u] = t < total;
            rr[u] = live[u] ? (uint32_t)(t / mb) : 0; blk[u] = live[u] ? (uint32_t)(t % mb) : 0;
            off[u] = 0; ntok[u] = 0;
            if (live[u]) { off[u] = __ldg(b.offsets + rr[u]); ntok[u] = __ldg(b.offsets + rr[u] + 1) - off[u]; }
        }
        if (BS == 16) {   // all token loads of the thread's UNR blocks in flight before the first hash
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const uint32_t nb = ntok[u] / 16;
                const uint32_t* p = b.tokens + off[u] + (size_t)blk[u] * 16;
                if (live[u] && blk[u] < nb) {
                    if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
                        const uint4* q = reinterpret_cast<const uint4*>(p);
#pragma unroll
                        for (int i = 0; i < 4; ++i) { uint4 x = __ldg(q + i); w[u][4 * i] = x.x; w[u][4 * i + 1] = x.y; w[u][4 * i + 2] = x.z; w[u][4 * i + 3] = x.w; }
                    } else {
#pragma unroll
                        for (int i = 0; i < 16; ++i) w[u][i] = __ldg(p + i);
                    }
                }
            }
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            if (!live[u]) continue;
            const uint32_t nb = ntok[u] / bs;
            SearchRec* rec = a.recs + (uint64_t)b.hash_base + rr[u];
            if (blk[u] == 0) rec->ntok = ntok[u];
            if (blk[u] < nb) {
                const uint64_t h = BS == 16 ? xxh3_16words(w[u], kSeed) : xxh3_words(b.tokens + off[u] + (size_t)blk[u] * bs, bs, kSeed);
                a.hashes[((uint64_t)b.hash_base + rr[u]) * mb + blk[u]] = h;
                if (blk[u] == 0) rec->h0 = h;
                if (blk[u] == min(a.pf_jump, nb - 1)) rec->h1 = h;
                if (a.pf_slots && (blk[u] == 0 || blk[u] == min(a.pf_jump, nb - 1)))
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const Slot*>(a.pf_slots) + (slot_hash(blk[u], h) & a.pf_mask)));
            }
        }
    }
    __threadfence();
    __syncthreads();
    // groups of 256 requests = 256·mb consecutive slots; this CTA's slots [t0, t1] touch groups g_first..g_last (one, unless mb is odd or tiny)
    const uint64_t gsz = 256ull * mb;
    const uint64_t t1 = (t0 + 256ull * UNR < total ? t0 + 256ull * UNR : total) - 1;
    const uint32_t g_first = (uint32_t)(t0 / gsz), g_last = (uint32_t)(t1 / gsz);
    for (uint32_t g = g_first; g <= g_last; ++g) {
        if (threadIdx.x == 0) {
            const uint64_t lo = (uint64_t)g * gsz, hi = lo + gsz < total ? lo + gsz : total;    // the group's slots [lo, hi)
            const uint32_t n_cta = (uint32_t)((hi - 1) / (256u * UNR) - lo / (256u * UNR)) + 1;
            uint32_t* cnt = a.group_count + (uint64_t)blockIdx.y * a.group_stride + g;
            const uint32_t old = atomicAdd(cnt, 1u);
            sm.last = old + 1 == n_cta;
            if (sm.last) *cnt = 0;                                                              // nobody else touches it until the next launch
        }
        __syncthreads();
        if (sm.last) {
            __threadfence();
            search2_body<false, true>(v, f, a, blockIdx.y, g * 256u, min(256u, b.n - g * 256u), sm, smem_ch);
        }
        __syncthreads();
    }
}

// ---- ONE launch, persistent CTAs: tokens streamed through a shared-memory ring by the copy engine, each CTA searches what it hashed ----
// What the measurements above ask for: the hash stream's bytes in flight must not depend on resident threads
// or on registers, and the search's chain of dependent round trips must be paid once per CTA, not once per request, tile or launch.
//   * The flattened list of tiles (a tile = the R = ⌊224 / max_blocks⌋ consecutive requests of one batch whose block slots fill one
//     14 KB stage) is dealt round-robin to the CTAs (tile g → CTA g mod grid); grid = resident CTAs (4 per SM).
//   * Warp 7 is the PRODUCER: per tile, lane j reads request j's offsets (one tile ahead of the ring), waits on the stage's `empty`
//     mbarrier, and issues ONE bulk copy (cp.async.bulk → UBLKCP, completion counted on the stage's `full` mbarrier) of the request's
//     whole blocks, global → stage slot j.  Three stages per CTA, all of them in flight whenever the consumers are ahead: up to 168 KB
//     per SM with no register and no thread waiting on them.  A request whose tokens are not 16 B aligned is copied by the producer
//     warp with plain loads instead.
//   * Warps 0-6 are CONSUMERS.  They read a stage TRANSPOSED: lane l of warp w takes the 16 B chunk l & 3 of blocks 32w + (l >> 2) +
//     8k, k = 0..3 — conflict-free LDS.128, after which the warp releases the stage — and does that chunk's XXH3 lane mix (each of
//     the four 16 B mixes of a 64 B input has its own secret words and is independent of the others); a 4-lane shuffle sum gives the
//     accumulator, lane l finishes block (l >> 2) + 8·(l & 3).  Hash rows, records and the L2 prefetch of the first two slots are as
//     in hash_blocks_kernel.  No CTA-wide barrier per tile: the warps drift.
//   * After ≤ 224 requests (or at the end of its tiles, or of a batch) the consumers meet on a named barrier and run search2_body on
//     them (a run of equally spaced tiles): the rows they read were written by the CTA's own threads (bar.sync + ld.global.cg).  Meanwhile the producer keeps the
//     ring full.
constexpr int kStStages = 3;
constexpr int kStConsumers = 224;                                   // 7 hashing warps; warp 7 feeds the ring
constexpr uint32_t kStStageBytes = kStConsumers * 64;               // 14 KB

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, uint32_t* err_flag) {
    uint32_t spins = 0;
    for (;;) {
        uint32_t ok;   // try_wait suspends the thread up to the hint (ns) while the phase is pending: few issue slots are spent spinning
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(bar), "r"(parity), "r"(2000u) : "memory");
        if (ok) return;
        if (++spins > (1u << 22)) { atomicExch(err_flag, 3u); return; }   // seconds: the other side never arrived — report, do not hang
    }
}
// the flattened tile list: tile = R consecutive requests of one batch
struct StPos { uint32_t y, r0; };
__device__ __forceinline__ StPos st_locate(const MultiArgs& a, uint32_t g, uint32_t R) {
    StPos t;
    if (a.uniform_n) { const uint32_t tpb = (a.uniform_n + R - 1) / R; t.y = g / tpb; t.r0 = (g - t.y * tpb) * R; }
    else {
        uint32_t y = 0, left = g;
        for (;; ++y) { const uint32_t tpb = (a.b[y].n + R - 1) / R; if (left < tpb || y + 1 >= a.count) break; left -= tpb; }
        t.y = y; t.r0 = left * R;
    }
    return t;
}
// `step` tiles further in the flattened list (the caller knows that tile exists)
__device__ __forceinline__ void st_next(const MultiArgs& a, StPos& t, uint32_t R, uint32_t step) {
    t.r0 += step * R;
    for (;;) {
        const uint32_t span = (a.b[t.y].n + R - 1) / R * R;       // the batch's tiles × R
        if (t.r0 < span) break;
        t.r0 -= span; ++t.y;
    }
}

// ---- the streaming kernel's own search: the same decisions as search2_body, organised around round trips -------------------------
// Timed inside the kernel (SMGX_STREAM_DBG=64) search2_body cost a CTA of 140 requests about as much in phase A as in phase B: not
// arithmetic, but chains of dependent round trips — fleet tables → record → slots in A; and in B one round (row → 31 probes → scan →
// record again) per PAIR of drains and warp, so 17 drains on 7 warps are two rounds.  Here
//   * the fleet tables and the derived fleet state are in shared memory from the start of the kernel;
//   * the consumers leave h0 / h1 / ntok of every hashed request in shared memory (no record in global memory at all);
//   * phase A is one thread per request: two probes in flight, classification, ONE argmax for whatever was decided;
//   * phase B issues every probe of up to 16 drains at once — (drain, position) pairs dealt over all 224 threads, results into a
//     shared-memory matrix — and only then replays the reference's ordered scan, one warp per drain, from that matrix: one round trip
//     for the whole CTA instead of one per pair;
//   * phase C (Multi entries, more than one jump) is the generic warp-cooperative search, as before.
constexpr int kStDrains = 16;
struct StreamSmem {
    int32_t slice[64];
    uint64_t load[64], ts[64];
    FleetDerived fd;
    uint64_t elig;
    uint64_t h0[kStConsumers], h1[kStConsumers];                  // of the requests hashed since the last search
    uint32_t ntok[kStConsumers];
    uint8_t qb[kStConsumers], qc[kStConsumers];
    uint32_t nb, nc;
    uint64_t dset[kStDrains][32];
    uint8_t dkind[kStDrains][32];                                  // 0 = no entry, 1 = Single, 2 = Multi
};

__device__ __forceinline__ void stream_search(const EventIndexView& v, const MultiArgs& a, const uint32_t y, const uint32_t r0, const uint32_t cnt,
                                              StreamSmem& sm, uint64_t* smem_ch) {
    if (a.dbg & 4) return;                                         // A/B: streaming only (no picks are written)
    constexpr int NT = kStConsumers;
    constexpr uint32_t NW = NT / 32;
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
    const BatchDesc& b = a.b[y];
    const bool cand_mode = b.cand != nullptr;
    const uint32_t mb = a.max_blocks;
    if (threadIdx.x == 0) { sm.nb = 0; sm.nc = 0; }
    search2_sync<NT>();                                            // the consumers' h0 / h1 / ntok are in shared memory, their hash rows in L2
    unsigned long long tr0 = 0, tr1 = 0, tr2 = 0;
    const bool trace = (a.dbg & 64) && threadIdx.x == 0 && blockIdx.x % 59 == 0;
    if (trace) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tr0));
    const uint64_t elig = sm.elig;
    auto finish = [&](uint32_t t, uint64_t win, uint32_t score) {  // argmax + store for request t of the segment (any single thread)
        int32_t out = sm.fd.min_load_idx;
        uint32_t branch = SMGX_BR_EVENT_MIN_LOAD, matched = 0;
        Cand c{false, 0, 0, -1};
        if (win) {
            while (win) { int id = __ffsll((long long)win) - 1; win &= win - 1; c.consider(sm.slice[id], sm.load[id], sm.ts[id]); }
            out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = score;
        }
        if (cand_mode) {
            smgx_shard_candidate sc;
            sc.score = c.have ? matched : 0; sc.local_idx = c.have ? (uint32_t)c.sl : 0xFFFFFFFFu; sc.load = c.ld; sc.tree_size = c.ts;
            b.cand[r0 + t] = sc;
        } else write_pick(b, r0 + t, out, branch, matched, sm.ntok[t]);
    };
    auto row_of = [&](uint32_t t) { return a.hashes + ((uint64_t)b.hash_base + r0 + t) * mb; };
    auto ld_hash = [&](const uint64_t* p) -> uint64_t { return (uint64_t)__ldcg(reinterpret_cast<const unsigned long long*>(p)); };

    // ---- phase A ----
    {
        const uint32_t t = threadIdx.x;
        enum { K_NONE, K_FIN, K_PICK };
        int kind = K_NONE;
        uint64_t win = 0;
        uint32_t score = 0, branch = 0;
        int32_t out = -1;
        if (t < cnt) {
            const uint32_t ntok = sm.ntok[t];
            const uint32_t nb = ntok / 16;
            if (!cand_mode && sm.fd.n_healthy == 0) { kind = K_PICK; out = -1; branch = SMGX_BR_NO_HEALTHY; }
            else if (!cand_mode && sm.fd.imbalanced) { kind = K_PICK; out = sm.fd.min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD; }
            else if (nb > mb) { atomicExch(a.err_flag, 1u); if (cand_mode) kind = K_FIN; else { kind = K_PICK; out = -1; branch = 255; } }
            else if (nb == 0 || v.n_workers == 0) kind = K_FIN;
            else if (nb - 1 > v.jump) sm.qc[atomicAdd(&sm.nc, 1u)] = (uint8_t)t;
            else {
                const uint32_t last = nb - 1;
                const uint64_t c0 = sm.h0[t], c1 = sm.h1[t];
                const uint32_t i0 = slot_hash(0, c0) & v.mask, i1 = slot_hash(last, c1) & v.mask;
                Slot s0 = load_slot(v.slots + i0), s1 = load_slot(v.slots + i1);          // both probes in flight together (L2-warm: prefetched at hash time)
                if (!finish_probe(v, 0, c0, i0, s0)) kind = K_FIN;                         // nothing cached at position 0 (:676-683)
                else if (s0.state != SLOT_SINGLE) sm.qc[atomicAdd(&sm.nc, 1u)] = (uint8_t)t;
                else if (s0.payload == 0 || last == 0) { kind = K_FIN; win = s0.payload & elig; score = nb; }
                else {
                    const bool f1 = finish_probe(v, last, c1, i1, s1);
                    if (f1 && s1.state != SLOT_SINGLE) sm.qc[atomicAdd(&sm.nc, 1u)] = (uint8_t)t;
                    else if (f1 && __popcll(s1.payload) == __popcll(s0.payload)) { kind = K_FIN; win = s0.payload & elig; score = nb; }   // count-only jump test (:720)
                    else sm.qb[atomicAdd(&sm.nb, 1u)] = (uint8_t)t;
                }
            }
        }
        if (kind == K_FIN) finish(t, win, score);
        else if (kind == K_PICK) write_pick(b, r0 + t, out, branch, 0, sm.ntok[t]);
    }
    search2_sync<NT>();
    if (trace) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tr1));

    // ---- phase B ----
    const uint32_t n_b = sm.nb;
    for (uint32_t base = 0; base < n_b; base += kStDrains) {
        const uint32_t chunk = min((uint32_t)kStDrains, n_b - base);
        for (uint32_t idx = threadIdx.x; idx < chunk * 32; idx += NT) {          // every probe of the chunk's drains at once
            const uint32_t d = idx >> 5, p = idx & 31;
            const uint32_t t = sm.qb[base + d];
            const uint32_t nb = sm.ntok[t] / 16;
            uint8_t kind = 0;
            uint64_t set = 0;
            if (p < nb) {
                const uint64_t h = ld_hash(row_of(t) + p);
                const uint32_t i = slot_hash(p, h) & v.mask;
                Slot sl = load_slot(v.slots + i);
                if (finish_probe(v, p, h, i, sl)) { kind = sl.state == SLOT_SINGLE ? 1 : 2; set = sl.payload; }
            }
            sm.dset[d][p] = set; sm.dkind[d][p] = kind;
        }
        search2_sync<NT>();
        for (uint32_t d = wic; d < chunk; d += NW) {                                // the ordered scan with its retain guard, from the matrix
            const uint32_t t = sm.qb[base + d];
            const uint32_t nb = sm.ntok[t] / 16;
            const int last = (int)nb - 1;
            const uint8_t kd = sm.dkind[d][lane];
            const uint64_t pl = sm.dset[d][lane];
            const bool found = kd != 0, single = kd == 1;
            uint64_t active = shfl64(pl, 0);                                         // phase A saw a Single entry at position 0
            const bool in_range = lane >= 1 && lane <= last;
            const uint32_t pc = single ? (uint32_t)__popcll(pl) : 0;
            uint64_t last_set = 0;
            uint32_t last_score = 0;
            bool bail = __shfl_sync(FULL, (int)kd, 0) != 1;
            unsigned remaining = __ballot_sync(FULL, in_range);
            while (!bail && remaining && active) {
                const uint32_t nact = (uint32_t)__popcll(active);
                const bool noop = single && pc >= nact;                              // retain guard (:611, :641)
                const unsigned bm = __ballot_sync(FULL, in_range && !noop) & remaining;
                if (!bm) break;
                const int k = __ffs((int)bm) - 1;
                if (!__shfl_sync(FULL, (int)found, k)) {                             // missing entry drains everything (:598-604)
                    const uint64_t e = active & elig;
                    if (e) { last_set = e; last_score = (uint32_t)k; }
                    active = 0;
                    break;
                }
                if (!__shfl_sync(FULL, (int)single, k)) { bail = true; break; }
                const uint64_t ws = shfl64(pl, k);
                if ((uint32_t)__popcll(ws) < nact) {
                    const uint64_t e = active & ~ws & elig;
                    if (e) { last_set = e; last_score = (uint32_t)k; }
                    active &= ws;
                }
                remaining &= ~((2u << k) - 1u);
            }
            if (lane == 0) {
                if (bail) sm.qc[atomicAdd(&sm.nc, 1u)] = (uint8_t)t;
                else {
                    uint64_t win = active & elig;
                    uint32_t score = nb;
                    if (!win) { win = last_set; score = last_score; }
                    finish(t, win, score);
                }
            }
        }
        search2_sync<NT>();
    }
    if (trace) {
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tr2));
        printf("cta %u n %u: phase A %llu ns, phase B %llu ns (nb %u nc %u)\n", blockIdx.x, cnt, tr1 - tr0, tr2 - tr1, sm.nb, sm.nc);
    }

    // ---- phase C: generic search ----
    const uint32_t n_c = sm.nc;
    uint64_t* row = smem_ch + (size_t)wic * mb;
    for (uint32_t q = wic; q < n_c; q += NW) {
        const uint32_t t = sm.qc[q];
        const uint32_t nb = sm.ntok[t] / 16;
        const uint64_t* ch = row_of(t);
        for (uint32_t i = lane; i < nb; i += 32) row[i] = ld_hash(ch + i);
        __syncwarp();
        const SlowResult sr = slow_search_inline<true>(v, row, (int)nb, lane, elig);
        if (lane == 0) finish(t, sr.winset, sr.score);
        __syncwarp();
    }
    search2_sync<NT>();
}

__global__ void __launch_bounds__(256, 4) event_stream_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a,
                                                              const uint32_t n_tiles) {
    extern __shared__ __align__(128) uint8_t st_dyn[];            // [3 stages × 14 KB][phase C rows: 7 × max_blocks u64][full[3], empty[3] mbarriers]
    __shared__ StreamSmem sm;
    const uint32_t mb = a.max_blocks;
    const uint32_t R = (uint32_t)kStConsumers / mb;               // requests per tile (launcher: 1 ≤ max_blocks ≤ 32)
    uint64_t* smem_ch = reinterpret_cast<uint64_t*>(st_dyn + kStStages * kStStageBytes);
    uint64_t* bars = smem_ch + 7 * mb;
    const uint32_t stage0 = smem_addr(st_dyn), full0 = smem_addr(bars), empty0 = full0 + 8 * kStStages;
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStStages; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(full0 + 8 * s), "r"(1));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(empty0 + 8 * s), "r"(kStConsumers / 32));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        sm.fd = *f.derived; sm.elig = f.elig[0];
    }
    if (threadIdx.x < 64) {
        const bool ok = threadIdx.x < v.n_workers;
        sm.slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        sm.load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        sm.ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    __syncthreads();
    // this CTA's tiles: one contiguous run of the flattened list (its requests are then contiguous inside every batch, which is what the
    // search's request = first + thread mapping needs).  Dealing the tiles round-robin instead — every CTA sweeping the same moving window
    // of the token buffers, like the stand-alone hash kernel's grid — was measured and streams no faster.
    const uint32_t G = 1;
    const uint32_t q_ = n_tiles / gridDim.x, rem_ = n_tiles % gridDim.x;
    const uint32_t g_n = q_ + (blockIdx.x < rem_ ? 1u : 0u);
    StPos pos = st_locate(a, blockIdx.x * q_ + min(blockIdx.x, rem_), R);

    if (wic == kStConsumers / 32) {
        // ---- producer warp: lane j (+32, +64 …) owns request slot j of every tile; the offsets are fetched one tile ahead of the copies ----
        const int n_u = (int)((R + 31) / 32);
        uint64_t pol_stream;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_stream));
        uint32_t o_lo[7], o_hi[7];                                  // offsets[r], offsets[r + 1] of this lane's requests of the NEXT tile to issue
        auto fetch = [&](const StPos& t) {
            const BatchDesc& b = a.b[t.y];
            const uint32_t cnt = min(R, b.n - t.r0);
#pragma unroll
            for (int u = 0; u < 7; ++u) {
                if (u >= n_u) break;
                const uint32_t j = (uint32_t)lane + 32u * u;
                o_lo[u] = 0; o_hi[u] = 0;
                if (j < cnt) { o_lo[u] = __ldg(b.offsets + t.r0 + j); o_hi[u] = __ldg(b.offsets + t.r0 + j + 1); }
            }
        };
        if (g_n) fetch(pos);
        for (uint32_t k = 0; k < g_n; ++k) {
            const BatchDesc& b = a.b[pos.y];
            const uint32_t cnt = min(R, b.n - pos.r0);
            const uint32_t s = k % kStStages, full = full0 + 8 * s;
            bool any_slow = false;
            uint32_t tx = 0;                                        // bytes the copy engine will deliver
            uint32_t bytes[7];
            const uint32_t* src[7];
#pragma unroll
            for (int u = 0; u < 7; ++u) {
                if (u >= n_u) break;
                const uint32_t j = (uint32_t)lane + 32u * u;
                const uint32_t nb = (o_hi[u] - o_lo[u]) / 16;
                bytes[u] = (j < cnt && nb <= mb) ? nb * 64 : 0;    // longer than max_blocks: search2_body flags the request, nothing is hashed
                src[u] = b.tokens + o_lo[u];
                const bool slow = bytes[u] && (reinterpret_cast<uintptr_t>(src[u]) & 15) != 0;
                any_slow = any_slow || slow;
                if (!slow) tx += bytes[u]; else bytes[u] |= 0x80000000u;
            }
            const StPos cur = pos;
            if (k + 1 < g_n) { st_next(a, pos, R, G); fetch(pos); }                            // in flight while this tile waits for its stage
            any_slow = __any_sync(FULL, any_slow);
            tx = __reduce_add_sync(FULL, tx);
            mbar_wait(empty0 + 8 * s, ((k / kStStages) & 1) ^ 1, a.err_flag);   // the consumers have read the stage's previous tile
            if (any_slow) {                                         // requests whose tokens are not 16 B aligned: plain loads by the whole warp
#pragma unroll 1
                for (uint32_t j = 0; j < cnt; ++j) {
                    const uint32_t off = __ldg(b.offsets + cur.r0 + j), ntok = __ldg(b.offsets + cur.r0 + j + 1) - off;
                    const uint32_t nb = ntok / 16;
                    const uint32_t* sp = b.tokens + off;
                    if (nb == 0 || nb > mb || (reinterpret_cast<uintptr_t>(sp) & 15) == 0) continue;
                    uint32_t* dst = reinterpret_cast<uint32_t*>(st_dyn + s * kStStageBytes + j * mb * 64);
                    for (uint32_t i = lane; i < nb * 16; i += 32) dst[i] = __ldg(sp + i);
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the stage's next fill is an async-proxy write
                __syncwarp();
            }
            if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full), "r"(tx) : "memory");
            __syncwarp();
#pragma unroll
            for (int u = 0; u < 7; ++u) {
                if (u >= n_u) break;
                const uint32_t j = (uint32_t)lane + 32u * u;
                if (bytes[u] && !(bytes[u] & 0x80000000u)) {
                    if (a.dbg & 128)   // A/B: tokens without the evict-first hint
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                     ::"r"(stage0 + s * kStStageBytes + j * mb * 64), "l"(src[u]), "r"(bytes[u]), "r"(full) : "memory");
                    else               // tokens are read once: evict-first, so that the stream does not push the prefetched index slots out of L2
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                                     ::"r"(stage0 + s * kStStageBytes + j * mb * 64), "l"(src[u]), "r"(bytes[u]), "r"(full), "l"(pol_stream) : "memory");
                }
            }
        }
        return;
    }

    // ---- consumer warps ----
    // this lane's chunk of a 64 B block: XXH3 17..128-byte path, len 64 — chunk 0 ↔ secret 0, 1 ↔ 32, 2 ↔ 48, 3 ↔ 16
    const int c = lane & 3;
    const uint64_t sec_lo = c == 0 ? sec64c<0>() : c == 1 ? sec64c<32>() : c == 2 ? sec64c<48>() : sec64c<16>();
    const uint64_t sec_hi = c == 0 ? sec64c<8>() : c == 1 ? sec64c<40>() : c == 2 ? sec64c<56>() : sec64c<24>();
    const uint64_t k_lo = sec_lo + kSeed, k_hi = sec_hi - kSeed;
    const uint32_t sb = 32u * (uint32_t)wic + (uint32_t)(lane >> 2) + 8u * (uint32_t)c;   // the slot this lane finishes: request sb / mb, block sb % mb
    const uint32_t my_j = sb / mb, my_blk = sb - my_j * mb;
    const uint32_t lds_off = (32u * wic + (lane >> 2)) * 64u + c * 16u;

    uint32_t seg_y = 0, seg_r0 = 0, seg_cnt = 0;                                           // hashed, not yet searched
    // the offsets of this lane's request are fetched one tile ahead
    uint32_t off = 0, ntok = 0;
    if (g_n && my_j < min(R, a.b[pos.y].n - pos.r0)) { off = __ldg(a.b[pos.y].offsets + pos.r0 + my_j); ntok = __ldg(a.b[pos.y].offsets + pos.r0 + my_j + 1) - off; }
    uint32_t k = 0;
    while (k < g_n) {
    // the hot loop: tiles of one segment; the search call sits outside it, so that nothing of the loop's state lives on the stack
    bool flush = false;
    do {
        const BatchDesc& b = a.b[pos.y];
        const uint32_t cnt = min(R, b.n - pos.r0), r0 = pos.r0, y = pos.y;
        const uint32_t s = k % kStStages;
        const uint32_t cur_ntok = ntok;
        StPos nx = pos;
        const bool more = k + 1 < g_n;
        uint32_t nx_cnt = 0;
        if (more) {
            st_next(a, nx, R, G);
            nx_cnt = min(R, a.b[nx.y].n - nx.r0);
            if (my_j < nx_cnt) { off = __ldg(a.b[nx.y].offsets + nx.r0 + my_j); ntok = __ldg(a.b[nx.y].offsets + nx.r0 + my_j + 1) - off; }
        }
        mbar_wait(full0 + 8 * s, (k / kStStages) & 1, a.err_flag);
        uint64_t acc = 0;
        {
            const uint8_t* base = st_dyn + s * kStStageBytes + lds_off;
            uint4 x[4];
#pragma unroll
            for (int rr = 0; rr < 4; ++rr) x[rr] = *reinterpret_cast<const uint4*>(base + rr * 8 * 64);
            // release the stage only once the four loads have RETURNED (the address depends on their data: a scoreboard wait, three instructions)
            uint32_t dep;
            asm volatile("and.b32 %0, %1, 0;" : "=r"(dep) : "r"(x[0].x | x[1].x | x[2].x | x[3].x));
            __syncwarp();
            if (lane == 0 && !(a.dbg & 1)) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * s + dep) : "memory");   // this warp has read the stage
#pragma unroll
            for (int rr = 0; rr < 4; ++rr) {
                uint64_t m = mul128_fold64(mk64(x[rr].x, x[rr].y) ^ k_lo, mk64(x[rr].z, x[rr].w) ^ k_hi);
                m += shfl64_xor(m, 1);
                m += shfl64_xor(m, 2);
                if (c == rr) acc = m;
            }
        }
        if (my_j < cnt) {
            const uint32_t nb = cur_ntok / 16;
            const uint32_t r = r0 + my_j;
            const uint32_t st = seg_cnt + my_j;                     // the request's place in the segment being collected
            if (my_blk == 0) sm.ntok[st] = cur_ntok;
            if (nb <= mb && my_blk < nb) {
                const uint64_t h = avalanche(acc + 64ULL * P64_1);
                a.hashes[((uint64_t)b.hash_base + r) * mb + my_blk] = h;
                const uint32_t jb = min(a.pf_jump, nb - 1);
                if (my_blk == 0) sm.h0[st] = h;
                if (my_blk == jb) sm.h1[st] = h;
                if (a.pf_slots && (my_blk == 0 || my_blk == jb))
                    asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(reinterpret_cast<const Slot*>(a.pf_slots) + (slot_hash(my_blk, h) & a.pf_mask)));
            }
        }
        if (a.dbg & 1) { __syncwarp(); if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * s) : "memory"); }
        if (seg_cnt == 0) { seg_y = y; seg_r0 = r0; }
        seg_cnt += cnt;
        flush = !more || nx.y != seg_y || seg_cnt + nx_cnt > (uint32_t)kStConsumers;
        pos = nx;
        ++k;
    } while (!flush);
    stream_search(v, a, seg_y, seg_r0, seg_cnt, sm, smem_ch);
    seg_cnt = 0;
    }
}

// ---- the same pick, TILED: one warp routes TILE consecutive requests of a batch -------------------------------------------------
// ncu on the warp-per-request kernel above: most of its warp instructions per request are not the XXH3 arithmetic — pipeline
// bookkeeping, descriptor fetches, probe/shuffle/pick logic and the store are paid once per REQUEST by a whole warp, and the kernel is
// issue-bound.  Here those costs are paid once per TILE:
//   phase 1  lane L fetches the offsets of request r0+L (one coalesced load for the tile); then, request by request, the warp streams the
//            2 KB of tokens (lane = block, the next request's 4×LDG.128 issued before the current one is hashed) and leaves the 32 content
//            hashes in a shared-memory row — ≈ 130 warp instructions per request, 106 of them hashing;
//   phase 2  lane L owns request r0+L: both jump destinations (positions 0 and last) probed by every lane at once — 2·TILE independent
//            32 B probes in flight per warp — count-only jump test, argmax, one coalesced store of the picks: ≈ 100 instructions per TILE;
//   phase 3  requests whose count test failed (stored prefix shorter than the request, Multi entries) are resolved one after another by
//            the generic warp-cooperative jump_search on their shared-memory row.
// Requirements (checked by the launcher, otherwise the warp-per-request kernel runs): ≤ 64 interned workers, block size 16, requests of
// ≤ 32 blocks with jump_size ≥ 31 (one jump), batches of equal size, plain picks (no shard candidates / load feedback).
// 16 B-aligned 64 B block of lane `lane` (loads issued, not consumed)
__device__ __forceinline__ void tile_load(const uint32_t* __restrict__ tokens, uint32_t off, uint32_t nb, int lane, uint32_t (&w)[16]) {
    if ((uint32_t)lane < nb) {
        const uint4* q4 = reinterpret_cast<const uint4*>(tokens + off + (size_t)lane * 16);
#pragma unroll
        for (int i = 0; i < 4; ++i) { uint4 t = __ldg(q4 + i); w[4 * i] = t.x; w[4 * i + 1] = t.y; w[4 * i + 2] = t.z; w[4 * i + 3] = t.w; }
    }
}

// DEPTH > 0: phase 1 streams the tokens through a per-warp shared-memory ring of DEPTH requests filled by cp.async (LDGSTS: 16 B per lane per
// instruction, [piece][lane] layout so that a lane reads its own 64 B back with four conflict-free LDS.128) — DEPTH × 2 KB per warp are in flight
// without holding a single register, which is what the register double buffer (DEPTH = 0) could not do: that variant keeps ≤ 2 requests in flight
// per warp and is latency-bound (few of the 64 warp slots busy).
template <int TILE, int MINB, int DEPTH>
__global__ void __launch_bounds__(128, MINB) event_tile_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a) {
    extern __shared__ uint64_t smem_ch[];   // [warps][TILE][32] hashes, then (DEPTH > 0) [warps][DEPTH][4][32] uint4 token stages
    __shared__ int32_t s_slice[64];
    __shared__ uint64_t s_load[64], s_ts[64];
    if (threadIdx.x < 64) {
        bool ok = threadIdx.x < v.n_workers;
        s_slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        s_load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        s_ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    uint64_t* ch = smem_ch + (size_t)wic * TILE * 32;
    const uint32_t n_healthy = f.derived->n_healthy, imbalanced = f.derived->imbalanced;
    const int32_t min_load_idx = f.derived->min_load_idx;
    const uint64_t elig = f.elig[0];
    const uint32_t n = a.uniform_n;
    const uint32_t tpb = (n + TILE - 1) / TILE, n_tiles = tpb * a.count;
    const uint32_t stride = gridDim.x * wpc;

#pragma unroll 1
    for (uint32_t t = blockIdx.x * wpc + wic; t < n_tiles; t += stride) {
        const uint32_t j = t / tpb, r0 = (t - j * tpb) * TILE;
        const BatchDesc& b = a.b[j];
        const uint32_t cnt = min((uint32_t)TILE, n - r0);
        uint32_t off = 0, ntok = 0;
        if ((uint32_t)lane < cnt) { off = __ldg(b.offsets + r0 + lane); ntok = __ldg(b.offsets + r0 + lane + 1) - off; }
        uint32_t nb = ntok >> 4;
        const bool too_long = nb > a.max_blocks;
        if (too_long) { nb = 0; atomicExch(a.err_flag, 1u); }
        const bool trivial = n_healthy == 0 || imbalanced;   // no index involvement: None / first min load (cache_aware.rs:653-655, :670)

        // ---- phase 1: hash the tile, request by request (lane = block), next request's loads in flight while this one is hashed ----
        if (!trivial) {
            // 16 B alignment of every request of the tile (warp-uniform): the pipelined loop issues LDG.128 only
            const bool aligned = (reinterpret_cast<uintptr_t>(b.tokens) & 15) == 0 && !__any_sync(FULL, (uint32_t)lane < cnt && (off & 3) != 0);
            if (aligned && DEPTH > 0) {
                uint4* ring = reinterpret_cast<uint4*>(smem_ch + (size_t)wpc * TILE * 32) + (size_t)wic * (DEPTH > 0 ? DEPTH : 1) * 128;
                auto issue = [&](uint32_t i) {   // request i of the tile → stage i % DEPTH; one commit group per call, empty when there is nothing to copy
                    if (i < cnt) {
                        const uint32_t off_i = __shfl_sync(FULL, off, (int)i), nb_i = __shfl_sync(FULL, nb, (int)i);
                        if ((uint32_t)lane < nb_i) {
                            const uint32_t* src = b.tokens + off_i + (size_t)lane * 16;
                            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(ring + (size_t)(i % (DEPTH > 0 ? DEPTH : 1)) * 128 + lane);
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + k * 512), "l"(src + k * 4) : "memory");
                        }
                    }
                    asm volatile("cp.async.commit_group;" ::: "memory");
                };
#pragma unroll
                for (int s0 = 0; s0 < DEPTH; ++s0) issue((uint32_t)s0);
#pragma unroll 1
                for (uint32_t i = 0; i < cnt; ++i) {
                    asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH > 0 ? DEPTH - 1 : 0) : "memory");   // groups complete in order: request i has landed
                    const uint32_t nb_i = __shfl_sync(FULL, nb, (int)i);
                    if ((uint32_t)lane < nb_i) {
                        const uint4* st = ring + (size_t)(i % (DEPTH > 0 ? DEPTH : 1)) * 128 + lane;
                        uint32_t w[16];
#pragma unroll
                        for (int k = 0; k < 4; ++k) { const uint4 t4 = st[k * 32]; w[4 * k] = t4.x; w[4 * k + 1] = t4.y; w[4 * k + 2] = t4.z; w[4 * k + 3] = t4.w; }
                        ch[i * 32 + lane] = xxh3_16words(w, kSeed);
                    }
                    issue(i + DEPTH);   // refill the stage this lane has just read (every lane touches only its own 64 B of a stage)
                }
                asm volatile("cp.async.wait_group 0;" ::: "memory");
            } else if (aligned) {
                uint32_t w0[16], w1[16];
                uint32_t off_i = __shfl_sync(FULL, off, 0), nb_i = __shfl_sync(FULL, nb, 0);
                tile_load(b.tokens, off_i, nb_i, lane, w0);
#pragma unroll 1
                for (uint32_t i = 0; i < cnt; i += 2) {
                    // request i (tokens in w0); issue request i+1 into w1 first
                    const uint32_t off_1 = __shfl_sync(FULL, off, (int)(i + 1) & 31), nb_1 = (i + 1 < cnt) ? __shfl_sync(FULL, nb, (int)(i + 1) & 31) : 0;
                    tile_load(b.tokens, off_1, nb_1, lane, w1);
                    if ((uint32_t)lane < nb_i) ch[i * 32 + lane] = xxh3_16words(w0, kSeed);
                    // request i+1 (tokens in w1); issue request i+2 into w0 first
                    const uint32_t off_2 = __shfl_sync(FULL, off, (int)(i + 2) & 31), nb_2 = (i + 2 < cnt) ? __shfl_sync(FULL, nb, (int)(i + 2) & 31) : 0;
                    tile_load(b.tokens, off_2, nb_2, lane, w0);
                    if ((uint32_t)lane < nb_1) ch[(i + 1) * 32 + lane] = xxh3_16words(w1, kSeed);
                    nb_i = nb_2;
                }
            } else {
#pragma unroll 1
                for (uint32_t i = 0; i < cnt; ++i) {
                    const uint32_t off_i = __shfl_sync(FULL, off, (int)i), nb_i = __shfl_sync(FULL, nb, (int)i);
                    if ((uint32_t)lane < nb_i) ch[i * 32 + lane] = hash_block<16>(b.tokens + off_i + (size_t)lane * 16, 16);
                }
            }
            __syncwarp();
        }

        // ---- phase 2: lane L decides request r0 + L ----
        int32_t out = -1;
        uint32_t branch = SMGX_BR_NO_HEALTHY, matched = 0;
        bool slow = false;
        const bool mine = (uint32_t)lane < cnt;
        if (mine) {
            if (n_healthy == 0) {
            } else if (imbalanced) { out = min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD; }
            else if (too_long) { branch = 255; }
            else {
                out = min_load_idx; branch = SMGX_BR_EVENT_MIN_LOAD;   // until an overlap is found
                if (nb > 0 && v.n_workers > 0) {
                    const int last = (int)nb - 1;
                    const uint64_t c0 = ch[lane * 32], c1 = ch[lane * 32 + last];
                    const uint32_t h0 = slot_hash(0, c0) & v.mask, h1 = slot_hash((uint32_t)last, c1) & v.mask;
                    Slot s0 = load_slot(v.slots + h0), s1 = load_slot(v.slots + h1);          // both probes in flight together
                    uint64_t win = 0;
                    if (finish_probe(v, 0, c0, h0, s0)) {
                        if (s0.state != SLOT_SINGLE) slow = true;
                        else if (s0.payload != 0) {
                            if (last == 0) win = s0.payload & elig;
                            else if (finish_probe(v, (uint32_t)last, c1, h1, s1) && s1.state == SLOT_SINGLE && __popcll(s1.payload) == __popcll(s0.payload)) win = s0.payload & elig;
                            else slow = true;   // count test failed (or a Multi entry): the generic search decides
                        }
                    }
                    if (win) {
                        Cand c{false, 0, 0, -1};
                        while (win) { int id = __ffsll((long long)win) - 1; win &= win - 1; c.consider(s_slice[id], s_load[id], s_ts[id]); }
                        out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = nb;
                    }
                }
            }
        }
        // ---- phase 3: the tile's slow requests, one after another, warp-cooperatively ----
        unsigned sm = __ballot_sync(FULL, slow);
        while (sm) {
            const int L = __ffs((int)sm) - 1;
            sm &= sm - 1;
            const int nb_L = (int)__shfl_sync(FULL, nb, L);
            const SlowResult sr = fused_slow_search<true>(&v, ch + L * 32, nb_L, lane, elig);
            if (lane == L) {
                uint64_t win = sr.winset;
                if (win) {
                    Cand c{false, 0, 0, -1};
                    while (win) { int id = __ffsll((long long)win) - 1; win &= win - 1; c.consider(s_slice[id], s_load[id], s_ts[id]); }
                    out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = sr.score;
                }
            }
        }
        if (mine) write_pick(b, r0 + lane, out, branch, matched, ntok);
        __syncwarp();   // the shared-memory rows are reused by the next tile
    }
}

// ---- the same pick, ONE THREAD per request, rare shapes queued for event_slow_kernel --------------------------------------------
// One warp per request (event_warp_kernel below) keeps 40 requests in flight per SM, and a full hit runs the whole warp's instruction
// stream for two useful lanes: that pick is bound by latency and instruction issue, not by bytes.  Here a CTA of 256 threads decides 256
// consecutive requests g (global index over the launch's batches: a CTA may straddle two batches) in two phases:
//   A  one THREAD per request: offsets, the fleet gate, the tokens of blocks 0 and last (all eight 16 B loads issued before either hash),
//      both hashes, both probes in flight together, the count-only jump test (event_tree.rs:720).  A block's content hash depends on
//      that block alone, so a full hit or a novel request reads 128 B of tokens.  A failed count test goes onto a shared-memory queue
//      together with what both probes found;
//   B  each warp serves four queued drains at a time, 8 lanes each, in segments of 8 positions: a lane reads and hashes one block and
//      looks it up in the tag array (tag_sector / tag_finish: a slot is read only where the tag matches), the queued probe of `last`
//      stands in for its block, and the ordered scan is replayed over the segment.  A drain stops at the segment where the scan stops
//      (a missing position, an empty active set), so a partial hit reads the blocks up to its stored prefix's end and not the rest;
//      its slot then takes the next queued drain.
// What needs the rolling prefix hashes or more than one jump (Multi entries, > 32 blocks, jump_size < blocks − 1) is pushed onto a device
// queue, at most once per request (from A or from B), and finished by event_slow_kernel right behind.  That kernel is launched only when
// such a request is possible: the index holds a Multi entry, or the launch allows more than 32 blocks or more than one jump (MultiArgs.skip_slow).
struct SimpleLoc { uint32_t j, r; };
__device__ __forceinline__ SimpleLoc simple_locate(const MultiArgs& a, uint32_t g) {
    SimpleLoc l;
    if (a.uniform_n) { l.j = g / a.uniform_n; l.r = g - l.j * a.uniform_n; }
    else { l.j = 0; while (l.j + 1 < a.count && a.b[l.j + 1].hash_base <= g) ++l.j; l.r = g - a.b[l.j].hash_base; }
    return l;
}

// a failed count test: request, token range, the probes of blocks 0 and last, the run-arena anchor of block 0's entry
struct LaneDrain { uint32_t g, off, ntok, f1; uint64_t p0, p1; uint32_t anchor; };

// queues request g for event_slow_kernel; a launch that skipped that kernel (a.skip_slow) reports it as an internal error instead (a bit
// OR-ed into err_flag, as the over-the-cap 1 of these kernels is, so that neither clears the other)
__device__ __forceinline__ void push_slow(const MultiArgs& a, uint32_t* slow_queue, uint32_t g) {
    if (a.skip_slow) atomicOr(a.err_flag, kErrNoSlowKernel);
    else slow_queue[2 + atomicAdd(slow_queue, 1u)] = g;
}

__global__ void __launch_bounds__(256, 4) event_lane_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a,
                                                            uint32_t* __restrict__ slow_queue) {
    __shared__ int32_t s_slice[64];
    __shared__ uint64_t s_load[64], s_ts[64];
    __shared__ LaneDrain s_q[256];
    __shared__ uint32_t s_n, s_head;   // queued drains; the next drain a free slot of phase B takes
    if (threadIdx.x < 64) {
        bool ok = threadIdx.x < v.n_workers;
        s_slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        s_load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        s_ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    if (threadIdx.x == 0) { s_n = 0; s_head = 32; }
    __syncthreads();
    const int32_t min_load_idx = f.derived->min_load_idx;
    const uint64_t elig = f.elig[0];
    auto to_slow = [&](uint32_t g) { push_slow(a, slow_queue, g); };

    // ---- phase A ----
    const uint32_t g = blockIdx.x * 256 + threadIdx.x;
    if (g < a.total) {
        const SimpleLoc loc = simple_locate(a, g);
        const BatchDesc& b = a.b[loc.j];
        const uint32_t off = __ldg(b.offsets + loc.r), ntok = __ldg(b.offsets + loc.r + 1) - off;
        const uint32_t nb = ntok >> 4;
        if (f.derived->n_healthy == 0) write_pick(b, loc.r, -1, SMGX_BR_NO_HEALTHY, 0, ntok);
        else if (f.derived->imbalanced) write_pick(b, loc.r, min_load_idx, SMGX_BR_IMBALANCED_MIN_LOAD, 0, ntok);
        else if (nb > a.max_blocks) { atomicOr(a.err_flag, 1u); write_pick(b, loc.r, -1, 255, 0, ntok); }
        else if (nb == 0 || v.n_workers == 0) finish_pick(b, loc.r, s_slice, s_load, s_ts, min_load_idx, 0, 0, ntok);
        else if (nb > 32 || nb - 1 > v.jump) to_slow(g);   // more than one jump / more blocks than lanes: the generic search
        else {
            const uint32_t last = nb - 1;
            uint32_t w0[16], w1[16];
            load_block16_pair(b.tokens + off, b.tokens + off + (size_t)last * 16, w0, w1);
            const uint64_t c0 = xxh3_16words(w0, kSeed), c1 = xxh3_16words(w1, kSeed);
            const uint32_t h0 = slot_hash(0, c0) & v.mask, h1 = slot_hash(last, c1) & v.mask;
            Slot s0 = load_slot(v.slots + h0), s1 = load_slot(v.slots + h1);   // both probes in flight together
            if (!finish_probe(v, 0, c0, h0, s0)) finish_pick(b, loc.r, s_slice, s_load, s_ts, min_load_idx, 0, 0, ntok);   // nothing cached at 0 (:676-683)
            else if (s0.state != SLOT_SINGLE) to_slow(g);
            else if (s0.payload == 0 || last == 0) finish_pick(b, loc.r, s_slice, s_load, s_ts, min_load_idx, s0.payload & elig, nb, ntok);
            else {
                const bool f1 = finish_probe(v, last, c1, h1, s1);
                if (f1 && s1.state != SLOT_SINGLE) to_slow(g);
                else if (f1 && __popcll(s1.payload) == __popcll(s0.payload))   // count-only jump test (:720)
                    finish_pick(b, loc.r, s_slice, s_load, s_ts, min_load_idx, s0.payload & elig, nb, ntok);
                else s_q[atomicAdd(&s_n, 1u)] = LaneDrain{g, off, ntok, (uint32_t)f1, s0.payload, s1.payload, s0.run};
            }
        }
    }
    __syncthreads();

    // ---- phase B: segments of 8 positions, four drains per warp round ----
    // Lanes 8d..8d+7 serve drain slot d; in a round, lane 8d+j reads, hashes and looks up position 1 + 8·seg + j of its slot's drain
    // (seg: the drain's next segment), the position `last` being phase A's probe carried in the queue.  The ordered scan is then replayed
    // over the segment from the scan state the slot's lanes carry (the active set, the latest drained set and its score).  A drain ends
    // where the scan ends: at a missing position (nothing after it can change the pick, event_tree.rs:598-604), when the active set is
    // empty, at an entry that needs the generic search, or once `last` is replayed; its slot then takes the next queued drain.
    const int lane = threadIdx.x & 31, sub = lane & 7, lead = lane & 24;
    const unsigned slot_bits = 0xffu << lead;
    const uint32_t n_d = s_n;
    uint32_t qi = (threadIdx.x >> 5) + 8u * (uint32_t)(lane >> 3);   // the first 32 drains spread over the warps; then s_head
    uint64_t active = qi < n_d ? s_q[qi].p0 : 0, last_set = 0;
    uint32_t last_score = 0, seg = 0, anchor = qi < n_d ? s_q[qi].anchor : kNil;
    while (__any_sync(FULL, qi < n_d)) {
        const bool live = qi < n_d;
        const LaneDrain& d = s_q[live ? qi : 0];
        const uint32_t last = live ? (d.ntok >> 4) - 1 : 0, pos = 1 + 8 * seg + (uint32_t)sub;
        const bool in_range = live && pos <= last;
        bool found = false;
        uint32_t reanchor = kNil;
        Slot sl{0, 0, SLOT_EMPTY, kNil, 0, 0};
        if (in_range && pos < last) {
            // the record the run layout puts at this position, loaded beside the tokens (neither depends on the hash): where it
            // is a live record of the key, it is the entry (event_index.h), and the tag walk and the cold slot are skipped
            const uint32_t ri = anchor + pos;
            uint4 ra = make_uint4(0, 0, SLOT_EMPTY, 0);
            uint2 rb = make_uint2(0, 0);
            if (ri < v.n_runs) {
                const uint4* q = reinterpret_cast<const uint4*>(v.runs + ri);
                ra = __ldg(q);
                rb = __ldg(reinterpret_cast<const uint2*>(q + 1));
            }
            uint32_t w[16];
            load_block16(a.b[simple_locate(a, d.g).j].tokens + d.off + (size_t)pos * 16, w);
            const uint64_t h = xxh3_16words(w, kSeed);
            if (mk64(ra.x, ra.y) == h && ra.z == pos && ra.w != SLOT_EMPTY) {
                found = true; sl.state = ra.w; sl.payload = mk64(rb.x, rb.y);
            } else {
                const uint32_t rep = tag_rep(pos, h);
                const TagCursor c = tag_sector(v, rep, slot_hash(pos, h) & v.mask);
                if (c.cand) sl = load_slot(v.slots + tag_slot(c));
                found = tag_finish(v, pos, h, rep, c, sl, sl);
                if (found && sl.run != kNil) reanchor = sl.run - pos;   // the run that holds this position, for the next segments
            }
        }
        __syncwarp();   // keeps the queued probe's shared-memory loads here, below the token load
        if (in_range && pos == last) { found = d.f1 != 0; sl.state = SLOT_SINGLE; sl.payload = d.p1; }
        {   // a slot's lanes that found their key outside the anchored run re-anchor the drain at the highest such position
            const unsigned rbits = __ballot_sync(FULL, reanchor != kNil) & slot_bits;
            const uint32_t ra = __shfl_sync(FULL, reanchor, rbits ? 31 - __clz((int)rbits) : lane);
            if (rbits) anchor = ra;
        }
        // drain_resolve's ballot loop, each slot on its own 8-bit field of the ballots
        const uint32_t cnt = (found && sl.state == SLOT_SINGLE) ? (uint32_t)__popcll(sl.payload) : 0;
        unsigned remaining = __ballot_sync(FULL, in_range) & slot_bits;
        bool bail = false;
        for (;;) {
            const uint32_t nact = (uint32_t)__popcll(active);
            const bool noop = found && sl.state == SLOT_SINGLE && cnt >= nact;   // retain guard (:611, :641)
            const unsigned bm = __ballot_sync(FULL, in_range && !noop) & remaining;
            if (!__any_sync(FULL, bm != 0)) break;
            const int k = bm ? __ffs((int)bm) - 1 : lane;
            const bool fk = __shfl_sync(FULL, (int)found, k) != 0;
            const uint32_t sk = __shfl_sync(FULL, sl.state, k);
            const uint64_t ws = shfl64(sl.payload, k);
            if (bm) {
                const uint32_t pk = 1 + 8 * seg + (uint32_t)(k & 7);
                if (!fk) {                                                         // missing entry drains everything (:598-604)
                    const uint64_t e = active & elig;
                    if (e) { last_set = e; last_score = pk; }
                    active = 0;
                } else if (sk != SLOT_SINGLE) bail = true;
                else if ((uint32_t)__popcll(ws) < nact) {
                    const uint64_t e = active & ~ws & elig;
                    if (e) { last_set = e; last_score = pk; }
                    active &= ws;
                }
                remaining = (bail || !active) ? 0u : remaining & ~((2u << k) - 1u);
            }
        }
        const bool done = live && (bail || !active || 8 * seg + 8 >= last);
        if (done && sub == 0) {
            if (bail) to_slow(d.g);
            else {
                uint64_t win = active & elig;
                uint32_t score = last + 1;
                if (!win) { win = last_set; score = last_score; }
                const SimpleLoc l = simple_locate(a, d.g);
                finish_pick(a.b[l.j], l.r, s_slice, s_load, s_ts, min_load_idx, win, score, d.ntok);
            }
            qi = atomicAdd(&s_head, 1u);
        }
        qi = __shfl_sync(FULL, qi, lead);
        if (done) {
            active = qi < n_d ? s_q[qi].p0 : 0; last_set = 0; last_score = 0; seg = 0; anchor = qi < n_d ? s_q[qi].anchor : kNil;
        } else ++seg;
    }
}

// The same pick with one WARP per request, for launches too small to give every SM a CTA of event_lane_kernel (a lone batch of a few
// thousand requests): ⌈requests / 8⌉ CTAs spread the work over all SMs, where the lane kernel's ⌈requests / 256⌉ would occupy a few.
// Lane p owns block p; lanes 0 and last hash their blocks and probe the two jump destinations, and only a failed count test makes lanes
// 1..last-1 read and hash theirs and look them up in the tag array for drain_resolve.  Rare shapes go to the same queue for event_slow_kernel.
__global__ void __launch_bounds__(256, 5) event_warp_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a,
                                                            uint32_t* __restrict__ slow_queue) {
    __shared__ int32_t s_slice[64];
    __shared__ uint64_t s_load[64], s_ts[64];
    if (threadIdx.x < 64) {
        bool ok = threadIdx.x < v.n_workers;
        s_slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        s_load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        s_ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint32_t g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (g >= a.total) return;
    const SimpleLoc loc = simple_locate(a, g);
    const BatchDesc& b = a.b[loc.j];
    const uint32_t off = __ldg(b.offsets + loc.r), ntok = __ldg(b.offsets + loc.r + 1) - off;
    const FleetDerived* fd = f.derived;
    int32_t out = -1;
    uint32_t branch = SMGX_BR_NO_HEALTHY, matched = 0;
    if (fd->n_healthy == 0) {
    } else if (fd->imbalanced) { out = fd->min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD; }
    else {
        const uint32_t nb = ntok >> 4;
        if (nb > a.max_blocks) { if (lane == 0) atomicOr(a.err_flag, 1u); branch = 255; }
        else {
            out = fd->min_load_idx; branch = SMGX_BR_EVENT_MIN_LOAD;   // until an overlap is found
            if (nb > 0 && v.n_workers > 0) {
                if (nb > 32 || nb - 1 > v.jump) {   // more than one jump / more blocks than lanes: the generic search
                    if (lane == 0) push_slow(a, slow_queue, g);
                    return;
                }
                const int last = (int)nb - 1;
                Slot sl{0, 0, SLOT_EMPTY, 0, 0};
                bool found = false;
                if (lane == 0 || lane == last) found = probe(v, (uint32_t)lane, hash_block<16>(b.tokens + off + (size_t)lane * 16, 16), sl);
                const uint64_t elig = f.elig[0];
                uint64_t win = 0;
                uint32_t score = 0;
                bool bail = false;
                if (__shfl_sync(FULL, (int)found, 0)) {
                    if (__shfl_sync(FULL, sl.state, 0) != SLOT_SINGLE) bail = true;   // Multi at position 0: needs the prefix hash
                    else {
                        const uint64_t active = shfl64(sl.payload, 0);
                        win = active & elig; score = nb;
                        if (last > 0 && active) {
                            const bool fl = __shfl_sync(FULL, (int)found, last) != 0;
                            const uint32_t stl = __shfl_sync(FULL, sl.state, last);
                            uint32_t count = 0;   // count_workers_at(last) (:555-574)
                            if (fl) { if (stl == SLOT_SINGLE) count = (uint32_t)__popcll(shfl64(sl.payload, last)); else bail = true; }
                            if (!bail && count != (uint32_t)__popcll(active)) {
                                if (lane >= 1 && lane < last) found = tag_probe(v, (uint32_t)lane, hash_block<16>(b.tokens + off + (size_t)lane * 16, 16), sl);
                                const DrainResult d = drain_resolve((int)nb, elig, lane, found, sl);
                                bail = d.bail; win = d.win; score = d.score;
                            }
                        }
                    }
                }
                if (bail) {
                    if (lane == 0) push_slow(a, slow_queue, g);
                    return;
                }
                if (win) {
                    Cand c{false, 0, 0, -1};
                    while (win) { int id = __ffsll((long long)win) - 1; win &= win - 1; c.consider(s_slice[id], s_load[id], s_ts[id]); }
                    out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = score;
                }
            }
        }
    }
    if (lane == 0) write_pick(b, loc.r, out, branch, matched, ntok);
}

// the queue of event_lane_kernel / event_warp_kernel: generic warp-cooperative search, one warp per queued request (hashes staged in a shared-memory row)
__global__ void __launch_bounds__(256) event_slow_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a,
                                                         uint32_t* __restrict__ slow_queue) {
    extern __shared__ uint64_t smem_ch[];
    __shared__ int32_t s_slice[64];
    __shared__ uint64_t s_load[64], s_ts[64];
    if (threadIdx.x < 64) {
        bool ok = threadIdx.x < v.n_workers;
        s_slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        s_load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        s_ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    uint64_t* ch = smem_ch + (size_t)wic * a.max_blocks;
    const uint32_t n_slow = slow_queue[0];
    const uint64_t elig = f.elig[0];
    const int32_t min_load_idx = f.derived->min_load_idx;
    for (uint32_t q = blockIdx.x * wpc + wic; q < n_slow; q += gridDim.x * wpc) {
        const uint32_t g = slow_queue[2 + q];
        const SimpleLoc loc = simple_locate(a, g);
        const BatchDesc& b = a.b[loc.j];
        const uint32_t off = __ldg(b.offsets + loc.r), ntok = __ldg(b.offsets + loc.r + 1) - off;
        const uint32_t nb = ntok >> 4;
        for (uint32_t blk = lane; blk < nb; blk += 32) ch[blk] = hash_block<16>(b.tokens + off + (size_t)blk * 16, 16);
        __syncwarp();
        const SlowResult sr = fused_slow_search<true>(&v, ch, (int)nb, lane, elig);
        int32_t out = min_load_idx;
        uint32_t branch = SMGX_BR_EVENT_MIN_LOAD, matched = 0;
        if (sr.winset) {
            uint64_t win = sr.winset;
            Cand c{false, 0, 0, -1};
            while (win) { int id = __ffsll((long long)win) - 1; win &= win - 1; c.consider(s_slice[id], s_load[id], s_ts[id]); }
            out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = sr.score;
        }
        if (lane == 0) write_pick(b, loc.r, out, branch, matched, ntok);
        __syncwarp();
    }
    // the last CTA out resets the count and the exit counter for the next launch on this lane; the counter sits at a fixed word, so a
    // launch of another size still finds it at zero (the entries need no reset: only [2, 2 + count) is read)
    __syncthreads();
    if (threadIdx.x == 0 && atomicAdd(slow_queue + 1, 1u) == gridDim.x - 1) { slow_queue[0] = 0; slow_queue[1] = 0; }
}

// L2 prefetch of a request's token range, two pipeline stages ahead of its use: PF = 1 one bulk prefetch per request issued by lane 0
// (cp.async.bulk.prefetch.L2 → UBLKPF.L2: the TMA unit walks the range, no register, no scoreboard), PF = 2 one CCTL.PF2 per lane
// (its own 64 B block), PF = 0 none.  The tokens are then read from L2 one iteration later, so a warp never holds a second request's
// tokens in registers while it works (the first version did, and the 16 extra live registers spilled around the slow-path call).
template <int PF>
__device__ __forceinline__ void fused_prefetch(const uint32_t* __restrict__ tokens, uint32_t off, uint32_t ntok, int lane) {
    if (PF == 1) {
        if (lane == 0 && ntok >= 16) {
            const uintptr_t lo = reinterpret_cast<uintptr_t>(tokens + off) & ~(uintptr_t)15;
            const uintptr_t hi = (reinterpret_cast<uintptr_t>(tokens + off + (ntok & ~15u)) + 15) & ~(uintptr_t)15;
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(lo), "r"((uint32_t)(hi - lo)) : "memory");
        }
    } else if (PF == 2) {
        for (uint32_t blk = lane; blk < (ntok >> 4); blk += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(tokens + off + (size_t)blk * 16));
    }
}

template <bool W1, int BS, int MINB, int PF>
__global__ void __launch_bounds__(256, MINB) event_fused_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a) {
    extern __shared__ uint64_t smem_ch[];
    __shared__ int32_t s_slice[64];
    __shared__ uint64_t s_load[64], s_ts[64];
    __shared__ uint32_t s_park[8][16];
    if (W1 && threadIdx.x < 64) {
        bool ok = threadIdx.x < v.n_workers;
        s_slice[threadIdx.x] = ok ? f.slice_of_id[threadIdx.x] : -1;
        s_load[threadIdx.x] = ok ? f.load_of_id[threadIdx.x] : 0;
        s_ts[threadIdx.x] = ok ? v.tree_sizes[threadIdx.x] : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, wic = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    uint64_t* ch = smem_ch + (size_t)wic * a.max_blocks;
    const uint32_t n_healthy = f.derived->n_healthy, imbalanced = f.derived->imbalanced;
    const int32_t min_load_idx = f.derived->min_load_idx;
    const uint64_t elig = W1 ? f.elig[0] : ((uint32_t)lane < v.words ? f.elig[lane] : 0ULL);
    const uint32_t S = gridDim.x * wpc;
    const uint32_t bs = BS ? (uint32_t)BS : a.block_size;

    // pipeline stages: A = request being processed, B = its successor (tokens already prefetched into L2), C = prefetched now, D = offsets loaded now
    FusedPos pA{0, 0};
    fused_advance(a, pA, blockIdx.x * wpc + wic);
    FusedPos pB = pA; fused_advance(a, pB, S);
    FusedPos pC = pB; fused_advance(a, pC, S);
    FusedPos pD = pC; fused_advance(a, pD, S);
    uint32_t offA = 0, endA = 0, offB = 0, endB = 0, offC = 0, endC = 0, offD = 0, endD = 0;
    if (pA.j < a.count) { offA = __ldg(a.b[pA.j].offsets + pA.r); endA = __ldg(a.b[pA.j].offsets + pA.r + 1); }
    if (pB.j < a.count) { offB = __ldg(a.b[pB.j].offsets + pB.r); endB = __ldg(a.b[pB.j].offsets + pB.r + 1); }
    if (pC.j < a.count) { offC = __ldg(a.b[pC.j].offsets + pC.r); endC = __ldg(a.b[pC.j].offsets + pC.r + 1); }
    if (PF && BS == 16 && pB.j < a.count) fused_prefetch<PF>(a.b[pB.j].tokens, offB, endB - offB, lane);

#pragma unroll 1
    while (pA.j < a.count) {
        if (PF && BS == 16 && pC.j < a.count) fused_prefetch<PF>(a.b[pC.j].tokens, offC, endC - offC, lane);
        if (pD.j < a.count) { offD = __ldg(a.b[pD.j].offsets + pD.r); endD = __ldg(a.b[pD.j].offsets + pD.r + 1); }

        // ---- request A ----
        const BatchDesc& b = a.b[pA.j];
        uint32_t ntok = endA - offA;
        const bool cand_mode = b.cand != nullptr;
        int32_t out = -1;
        uint32_t branch = SMGX_BR_NO_HEALTHY, matched = 0;
        Cand best{false, 0, 0, -1};
        const bool fb = a.fb_winsets != nullptr && !cand_mode;   // load feedback: emit (tied set, score), the in-order pass picks
        if (!cand_mode && n_healthy == 0) {
        } else if (!fb && !cand_mode && imbalanced) {
            out = min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD;
        } else {
            const uint32_t nb = bs ? ntok / bs : 0;
            if (nb > a.max_blocks) {
                if (lane == 0) atomicExch(a.err_flag, 1u);
                branch = 255;
                if (fb) {
                    const size_t gi = (size_t)b.hash_base + pA.r;
                    if ((uint32_t)lane < v.words) a.fb_winsets[gi * v.words + lane] = 0;
                    if (lane == 0) a.fb_scores[gi] = 0xFFFFFFFFu;
                }
            }
            else {
                uint64_t winset = 0;
                uint32_t score = 0;
                if (nb > 0 && v.n_workers > 0) {
                    uint64_t h = 0;
                    if (BS == 16) { if ((uint32_t)lane < nb) h = hash_block<16>(b.tokens + offA + (size_t)lane * 16, 16); }
                    bool slow = true;
                    if (W1 && BS == 16 && nb <= 32 && nb - 1 <= v.jump) {
                        // fast path: destinations are exactly {0, last}; lane p holds the hash of block p
                        const int last = (int)nb - 1;
                        Slot sl{0, 0, SLOT_EMPTY, 0, 0};
                        bool found = false;
                        if (lane == 0 || lane == last) found = probe(v, (uint32_t)lane, h, sl);
                        const bool f0 = __shfl_sync(FULL, (int)found, 0) != 0;
                        const uint32_t st0 = __shfl_sync(FULL, sl.state, 0);
                        if (!f0) slow = false;                                   // nothing cached at position 0: no scores (:676-683)
                        else if (st0 == SLOT_SINGLE) {
                            const uint64_t act = shfl64(sl.payload, 0);
                            if (act == 0) slow = false;
                            else if (last == 0) { slow = false; winset = act & elig; score = nb; }
                            else {
                                const bool fl = __shfl_sync(FULL, (int)found, last) != 0;
                                const uint32_t stl = __shfl_sync(FULL, sl.state, last);
                                const uint64_t pl = shfl64(sl.payload, last);
                                if (fl && stl == SLOT_SINGLE && __popcll(pl) == __popcll(act)) { slow = false; winset = act & elig; score = nb; }   // count-only jump test (:720)
                            }
                        }
                    }
                    if (slow) {
                        if (BS == 16) {
                            if ((uint32_t)lane < nb) ch[lane] = h;
                            for (uint32_t blk = lane + 32; blk < nb; blk += 32) ch[blk] = hash_block<16>(b.tokens + offA + (size_t)blk * 16, 16);
                        } else {
                            for (uint32_t blk = lane; blk < nb; blk += 32) ch[blk] = hash_block<0>(b.tokens + offA + (size_t)blk * bs, bs);
                        }
                        // The generic search is a real call: whatever is live across it would have to sit in the few callee-saved registers, and
                        // ptxas answers by keeping the whole pipeline state in local memory for EVERY iteration.  The state is warp-uniform, so it
                        // is parked in 64 B of shared memory around the call instead — the common path keeps it in registers.
                        if (lane == 0) {
                            volatile uint32_t* pk = s_park[wic];
                            pk[0] = pA.j; pk[1] = pA.r; pk[2] = pB.j; pk[3] = pB.r; pk[4] = pC.j; pk[5] = pC.r; pk[6] = pD.j; pk[7] = pD.r;
                            pk[8] = offB; pk[9] = endB; pk[10] = offC; pk[11] = endC; pk[12] = offD; pk[13] = endD; pk[14] = ntok;
                        }
                        __syncwarp();
                        const SlowResult sr = fused_slow_search<W1>(&v, ch, (int)nb, lane, elig);
                        winset = sr.winset; score = sr.score;
                        __syncwarp();
                        {
                            const volatile uint32_t* pk = s_park[wic];
                            pA.j = pk[0]; pA.r = pk[1]; pB.j = pk[2]; pB.r = pk[3]; pC.j = pk[4]; pC.r = pk[5]; pD.j = pk[6]; pD.r = pk[7];
                            offB = pk[8]; endB = pk[9]; offC = pk[10]; endC = pk[11]; offD = pk[12]; endD = pk[13]; ntok = pk[14];
                        }
                    }
                }
                if (fb) {
                    const size_t gi = (size_t)b.hash_base + pA.r;
                    if (W1) { if (lane == 0) a.fb_winsets[gi] = winset; }
                    else if ((uint32_t)lane < v.words) a.fb_winsets[gi * v.words + lane] = winset;
                    if (lane == 0) a.fb_scores[gi] = score;
                } else if (set_any<W1>(winset)) {
                    if (W1) {
                        uint64_t w = winset;
                        const int id0 = __ffsll((long long)w) - 1;
                        w &= w - 1;
                        best.have = true; best.sl = s_slice[id0]; best.ld = s_load[id0]; best.ts = s_ts[id0];
                        while (w) { int id = __ffsll((long long)w) - 1; w &= w - 1; best.consider(s_slice[id], s_load[id], s_ts[id]); }
                    } else best = warp_arg_best(v, f, winset, lane);
                    out = best.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = score;
                } else { out = min_load_idx; branch = SMGX_BR_EVENT_MIN_LOAD; }
            }
        }
        if (lane == 0) {
            if (cand_mode) {
                smgx_shard_candidate sc;
                sc.score = best.have ? matched : 0; sc.local_idx = best.have ? (uint32_t)best.sl : 0xFFFFFFFFu; sc.load = best.ld; sc.tree_size = best.ts;
                b.cand[pA.r] = sc;
            } else if (!fb || n_healthy == 0) write_pick(b, pA.r, out, branch, matched, ntok);
        }
        // rotate the pipeline
        pA = pB; offA = offB; endA = endB;
        pB = pC; offB = offC; endB = endC;
        pC = pD; offC = offD; endC = endD;
        fused_advance(a, pD, S);
    }
    if (a.done_flag) {   // mapped submission: picks were stored straight into pinned host memory — publish completion to the spinning caller
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            if (atomicAdd(a.done_counter, 1u) == gridDim.x - 1) {
                *a.done_counter = 0;
                __threadfence_system();
                asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(a.done_flag), "l"(a.done_value) : "memory");
            }
        }
    }
}

template <bool W1>
__global__ void find_matches_kernel(EventIndexView v, const uint64_t* __restrict__ hashes, uint32_t n, int early_exit, uint32_t* scores) {
    extern __shared__ uint64_t smem_ch[];
    const int lane = threadIdx.x & 31;
    for (uint32_t i = lane; i < n; i += 32) smem_ch[i] = hashes[i];
    __syncwarp();
    if (n == 0 || v.n_workers == 0) return;
    DumpSink<W1> sink{scores, lane};
    uint64_t surv = jump_search<W1>(v, smem_ch, (int)n, lane, sink, early_exit != 0);
    sink.on_event(n, surv);
}

__global__ void content_hashes_kernel(const uint32_t* __restrict__ tokens, uint32_t n_tokens, uint32_t bs, uint64_t* out) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nb = bs ? n_tokens / bs : 0;
    if (b < nb) out[b] = xxh3_words(tokens + (size_t)b * bs, bs, kSeed);
}

// convert_kv_block for a batch of KV events (kv_event_monitor.rs:592-597): block j carries token_ids[offs[j] .. offs[j+1]) — any length,
// also empty — and its content hash is XXH3-64(seed 1337) over their little-endian bytes.  One thread per block.
__global__ void content_hashes_ragged_kernel(const uint32_t* __restrict__ tokens, const uint32_t* __restrict__ offs, uint32_t n_blocks, uint64_t* out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n_blocks) out[j] = xxh3_words(tokens + offs[j], offs[j + 1] - offs[j], kSeed);
}

__global__ void fill_kernel(uint32_t* d, uint32_t value, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) d[i] = value;
}

// select_worker prologue on the device: one CTA, the fleet is at most a few thousand workers.
__global__ void __launch_bounds__(256) fleet_prepare_kernel(FleetRaw raw, FleetDerived* out, int32_t* slice_of_id, uint64_t* load_of_id,
                                                            unsigned long long* elig) {
    __shared__ uint64_t s_mn[256], s_mx[256], s_hl[256];
    __shared__ int32_t s_hidx[256], s_fh[256];
    __shared__ uint32_t s_nh[256];
    const int tid = threadIdx.x;
    for (uint32_t i = tid; i < raw.n_ids; i += 256) { slice_of_id[i] = -1; load_of_id[i] = 0; }
    for (uint32_t i = tid; i < raw.words; i += 256) elig[i] = 0;
    __syncthreads();
    uint64_t mn = ~0ULL, mx = 0, hl = ~0ULL;
    int32_t hidx = 0x7fffffff, fh = 0x7fffffff;
    uint32_t nh = 0;
    for (uint32_t i = tid; i < raw.n_slice; i += 256) {
        uint64_t load = raw.loads[i];
        mn = load < mn ? load : mn;      // min/max over ALL workers, healthy or not (cache_aware.rs:662-666)
        mx = load > mx ? load : mx;
        if ((raw.flags[i] & 3) == 3) {   // is_healthy() && circuit_breaker_can_execute()  (mod.rs:137-144)
            ++nh;
            fh = (int32_t)i < fh ? (int32_t)i : fh;
            if (load < hl || (load == hl && (int32_t)i < hidx)) { hl = load; hidx = (int32_t)i; }
            int32_t id = raw.id_of_slice[i];
            if (id >= 0 && (uint32_t)id < raw.n_ids) {
                atomicOr(&elig[id >> 6], 1ULL << (id & 63));
                if (!raw.has_dups) { slice_of_id[id] = (int32_t)i; load_of_id[id] = load; }
            }
        }
    }
    if (raw.has_dups) {
        // Two slice entries with the same URL map to the same indexer id: score_overlap (cache_aware.rs:795-818) scores BOTH indices
        // with the same (score, tree_size), so among them max_by_key keeps the lowest load and, on equal loads, the LAST index.
        // Pre-reduce per id in slice order (one thread: fleets are a few thousand entries and this runs once per fleet snapshot).
        __syncthreads();
        if (tid == 0)
            for (uint32_t i = 0; i < raw.n_slice; ++i) {
                if ((raw.flags[i] & 3) != 3) continue;
                const int32_t id = raw.id_of_slice[i];
                if (id < 0 || (uint32_t)id >= raw.n_ids) continue;
                if (slice_of_id[id] < 0 || raw.loads[i] <= load_of_id[id]) { slice_of_id[id] = (int32_t)i; load_of_id[id] = raw.loads[i]; }
            }
    }
    s_mn[tid] = mn; s_mx[tid] = mx; s_hl[tid] = hl; s_hidx[tid] = hidx; s_fh[tid] = fh; s_nh[tid] = nh;
    __syncthreads();
    for (int d = 128; d; d >>= 1) {
        if (tid < d) {
            s_mn[tid] = s_mn[tid + d] < s_mn[tid] ? s_mn[tid + d] : s_mn[tid];
            s_mx[tid] = s_mx[tid + d] > s_mx[tid] ? s_mx[tid + d] : s_mx[tid];
            if (s_hl[tid + d] < s_hl[tid] || (s_hl[tid + d] == s_hl[tid] && s_hidx[tid + d] < s_hidx[tid])) {
                s_hl[tid] = s_hl[tid + d]; s_hidx[tid] = s_hidx[tid + d];
            }
            s_fh[tid] = s_fh[tid + d] < s_fh[tid] ? s_fh[tid + d] : s_fh[tid];
            s_nh[tid] += s_nh[tid + d];
        }
        __syncthreads();
    }
    if (tid == 0) {
        FleetDerived d;
        uint64_t mn0 = s_mn[0] == ~0ULL ? 0 : s_mn[0], mx0 = s_mx[0];
        // min_load keeps the fold's UINT64_MAX start value for an empty slice: a worker-id shard with no workers must not lower the
        // fleet minimum shard_reduce_kernel takes over the shards' summaries (the gate, here and there, maps UINT64_MAX to 0 like :666)
        d.min_load = s_mn[0]; d.max_load = mx0;
        d.n_healthy = s_nh[0];
        d.min_load_idx = s_nh[0] ? s_hidx[0] : -1;
        d.first_healthy = s_nh[0] ? s_fh[0] : -1;
        d.min_healthy_load = s_nh[0] ? s_hl[0] : 0;
        // usize→f32 casts round to nearest-even; the product is an f32 multiply (no FMA contraction possible here)
        float fmax = __ull2float_rn(mx0), fmin = __ull2float_rn(mn0);
        d.imbalanced = ((mx0 - mn0) > raw.abs_threshold && fmax > __fmul_rn(fmin, raw.rel_threshold)) ? 1u : 0u;
        *out = d;
    }
}

}  // namespace

void launch_fleet_prepare(const FleetRaw& raw, FleetDerived* d_derived, int32_t* d_slice_of_id, uint64_t* d_load_of_id, uint64_t* d_elig,
                          cudaStream_t stream) {
    fleet_prepare_kernel<<<1, 256, 0, stream>>>(raw, d_derived, d_slice_of_id, d_load_of_id, reinterpret_cast<unsigned long long*>(d_elig));
    SMGX_CUDA(cudaGetLastError());
}

// 0 = pair, 1 = warp-per-request family, 2 = one launch (hash stream + last-arriver search), 3 = persistent streaming kernel;
// initialised from SMGX_EVENT_PATH (split | fused | hs | stream), switchable at run time for A/B runs and tests
static std::atomic<int> g_event_path{-1};
int event_path() {
    int v = g_event_path.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("SMGX_EVENT_PATH");
        const std::string s = e ? e : "";
        v = s == "split" ? 0 : s == "stream" ? 3 : s == "hs" ? 2 : 1;   // on H100 path 1 (the simple kernel) beats the pair by ≈ 14 %
        g_event_path.store(v, std::memory_order_relaxed);
    }
    return v;
}
bool event_select_fused() { return event_path() == 1; }
void set_event_select_fused(bool fused) { g_event_path.store(fused ? 1 : 0, std::memory_order_relaxed); }
void set_event_path(int path) { g_event_path.store(path < 0 || path > 3 ? 0 : path, std::memory_order_relaxed); }
static std::atomic<int> g_fused_minb{-1};
void set_fused_minb(int minb) { g_fused_minb.store(minb == 3 ? 3 : 4, std::memory_order_relaxed); }

// resident CTAs per SM the fused kernel is compiled for: 4 = 64 registers / 32 warps, 3 = 80 registers / 24 warps (SMGX_FUSED_MINB, A/B runs)
static int fused_minb() {
    int v = g_fused_minb.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("SMGX_FUSED_MINB");
        v = (e && e[0] == '3') ? 3 : 4;
        g_fused_minb.store(v, std::memory_order_relaxed);
    }
    return v;
}
static std::atomic<int> g_fused_pf{-1};
void set_fused_prefetch(int pf) { g_fused_pf.store(pf < 0 || pf > 2 ? 1 : pf, std::memory_order_relaxed); }
static int fused_pf() {   // SMGX_FUSED_PF=0|1|2 (A/B runs): L2 prefetch flavour, default 1 = bulk
    int v = g_fused_pf.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("SMGX_FUSED_PF");
        v = (e && e[0] >= '0' && e[0] <= '2') ? e[0] - '0' : 1;
        g_fused_pf.store(v, std::memory_order_relaxed);
    }
    return v;
}
static std::atomic<int> g_tile{-1};
static std::atomic<long long> g_tile_min_total{-1};   // < 0: tile × 4 × SMs (enough tiles to fill the GPU a few times over)
void set_fused_tile(int tile, long long min_total) {
    g_tile.store((tile == 0 || tile == 8 || tile == 16 || tile == 32) ? tile : 16, std::memory_order_relaxed);
    g_tile_min_total.store(min_total, std::memory_order_relaxed);
}
static int fused_tile() {   // SMGX_FUSED_TILE=0|8|16|32: requests per warp of the tiled kernel (0 = always the warp-per-request kernel)
    int v = g_tile.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("SMGX_FUSED_TILE");
        v = e ? atoi(e) : 16;
        if (v != 0 && v != 8 && v != 16 && v != 32) v = 16;
        g_tile.store(v, std::memory_order_relaxed);
    }
    return v;
}
static std::atomic<int> g_simple{-1};
void set_event_simple(int minb) { g_simple.store(minb, std::memory_order_relaxed); }
static bool event_lane_selected() {   // SMGX_EVENT_SIMPLE=0|4|5|6: 0 = do not use the lane / warp kernels, 4 / 5 / 6 = use them (the default)
    int v = g_simple.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("SMGX_EVENT_SIMPLE");
        v = e ? atoi(e) : 5;
        if (v != 0 && v != 4 && v != 5 && v != 6) v = 5;
        g_simple.store(v, std::memory_order_relaxed);
    }
    return v != 0;
}
// → the number of kernels launched: 1 when a.skip_slow (event_slow_kernel could get no request), else 2
static int launch_lane(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream, uint32_t* d_queue) {
    // one thread per request once the launch gives every SM a CTA of 256; below that (a lone batch of a few thousand requests) one warp per
    // request spreads the work over all SMs and answers sooner (measured on H100: 4096 requests, §5 of DESIGN.md)
    if (a.total >= 256u * (unsigned)sm_count) event_lane_kernel<<<(a.total + 255) / 256, 256, 0, stream>>>(ix, fleet, a, d_queue);
    else event_warp_kernel<<<(a.total + 7) / 8, 256, 0, stream>>>(ix, fleet, a, d_queue);
    SMGX_CUDA(cudaGetLastError());
    if (a.skip_slow) return 1;
    const size_t smem = (size_t)std::max<uint32_t>(a.max_blocks, 1) * 8 * 8;
    if (smem > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(event_slow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // one warp per queued request: ⌈total / 8⌉ CTAs would give every request a warp, two per SM are plenty for the rare shapes it gets
    const unsigned slow_grid = std::min<unsigned>((unsigned)sm_count * 2, std::max(1u, (a.total + 7) / 8));
    event_slow_kernel<<<slow_grid, 256, smem, stream>>>(ix, fleet, a, d_queue);
    SMGX_CUDA(cudaGetLastError());
    return 2;
}

static std::atomic<int> g_tile_depth{-1};
void set_tile_depth(int d) { g_tile_depth.store(d, std::memory_order_relaxed); }
static int tile_depth() {   // SMGX_TILE_DEPTH=0|4|8: cp.async ring depth of the tiled kernel's token stream (0 = register double buffer)
    int v = g_tile_depth.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("SMGX_TILE_DEPTH");
        v = e ? atoi(e) : 0;   // measured: the ring is slower than the register double buffer
        if (v != 0 && v != 4 && v != 8) v = 0;
        g_tile_depth.store(v, std::memory_order_relaxed);
    }
    return v;
}
template <int TILE>
static void launch_tile(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream) {
    using K = void (*)(EventIndexView, FleetView, MultiArgs);
    const int minb = fused_minb(), depth = tile_depth();
    K k = depth == 8 ? (K)event_tile_kernel<TILE, 4, 8> : depth == 4 ? (K)event_tile_kernel<TILE, 4, 4>
        : minb == 3 ? (K)event_tile_kernel<TILE, 4, 0> : (K)event_tile_kernel<TILE, 5, 0>;
    const int wpc = 4;
    const size_t smem = (size_t)wpc * TILE * 32 * 8 + (size_t)wpc * depth * 2048;
    if (smem + 2048 > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // + the kernel's static arrays
    static thread_local int occ_cache[3][2] = {};
    int& occ = occ_cache[depth == 8 ? 2 : depth == 4 ? 1 : 0][minb == 3 ? 1 : 0];
    if (!occ) SMGX_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, wpc * 32, smem));
    const unsigned n_tiles = ((a.uniform_n + TILE - 1) / TILE) * a.count;
    const unsigned persistent = (unsigned)sm_count * (unsigned)std::max(occ, 1);
    k<<<std::max(1u, std::min(persistent, (n_tiles + wpc - 1) / wpc)), wpc * 32, smem, stream>>>(ix, fleet, a);
}

template <bool W1, int BS>
static void launch_fused(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream) {
    using K = void (*)(EventIndexView, FleetView, MultiArgs);
    const int minb = fused_minb(), pf = fused_pf();
    K k = minb == 3 ? (pf == 0 ? (K)event_fused_kernel<W1, BS, 3, 0> : pf == 2 ? (K)event_fused_kernel<W1, BS, 3, 2> : (K)event_fused_kernel<W1, BS, 3, 1>)
                    : (pf == 0 ? (K)event_fused_kernel<W1, BS, 4, 0> : pf == 2 ? (K)event_fused_kernel<W1, BS, 4, 2> : (K)event_fused_kernel<W1, BS, 4, 1>);
    const size_t per_warp = (size_t)std::max<uint32_t>(a.max_blocks, 1) * 8;
    int wpc = 8;
    while (wpc > 1 && per_warp * wpc > 64 * 1024) wpc >>= 1;
    const size_t smem = per_warp * wpc;
    if (smem > 200 * 1024) throw Error(SMGX_INVALID_ARGUMENT, "request too long for the per-warp scratch (max_tokens_per_request)");
    if (smem > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    static thread_local int occ_cache[3][2][2][2][4] = {};   // [pf][minb][W1][BS16][log2 wpc] for the common small-smem case
    int occ = 0;
    int& slot = occ_cache[pf][minb == 3 ? 1 : 0][W1 ? 1 : 0][BS == 16 ? 1 : 0][wpc == 8 ? 3 : wpc == 4 ? 2 : wpc == 2 ? 1 : 0];
    if (smem <= 4096 && slot) occ = slot;
    else {
        SMGX_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, wpc * 32, smem));
        if (smem <= 4096) slot = occ;
    }
    const unsigned persistent = (unsigned)sm_count * (unsigned)std::max(occ, 1);
    const unsigned need = (a.total + wpc - 1) / wpc;
    k<<<std::max(1u, std::min(persistent, need)), wpc * 32, smem, stream>>>(ix, fleet, a);
}

// Which implementation serves a launch.  SMGX_EVENT_PATH / smgx_set_event_path:
//   split                            hash stream kernel + balanced search kernel — the hash kernel is a pure bandwidth kernel (2048 resident
//                                    threads per SM), the search works on 24 B + probes per request; multi-batch calls pipeline the
//                                    two over two stream lanes (smgx.cu: enqueue_split_pipelined)
//   fused (default for plain picks)  one kernel per launch (simple / tiled / warp-per-request pipelined: see the kernels above).  Mapped
//                                    (zero-copy) submissions and load-feedback batches always run the warp-per-request fused kernel: they
//                                    need its completion word / tied-set outputs.
static bool needs_fused_kernel(const MultiArgs& a) { return a.done_flag != nullptr || a.fb_winsets != nullptr; }
bool event_launch_is_split(const MultiArgs& a) { return !event_select_fused() && !needs_fused_kernel(a); }

void launch_event_hash(const MultiArgs& a, int sm_count, cudaStream_t stream, uint64_t* launches) {
    uint32_t max_n = 0;
    for (uint32_t j = 0; j < a.count; ++j) max_n = std::max(max_n, a.b[j].n);
    if (!max_n || !a.block_size) return;
    // K2b hashes: one thread per block slot, capped at a few waves (grid-stride beyond that)
    uint64_t threads = (uint64_t)max_n * a.max_blocks;
    unsigned gx = (unsigned)std::min<uint64_t>((threads + 255) / 256, (uint64_t)sm_count * 64);
    if (a.block_size == 16) hash_blocks_kernel<16><<<dim3(std::max(1u, gx), a.count), 256, 0, stream>>>(a);
    else hash_blocks_kernel<0><<<dim3(std::max(1u, gx), a.count), 256, 0, stream>>>(a);
    SMGX_CUDA(cudaGetLastError());
    ++*launches;
}
void launch_event_search(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream, uint64_t* launches) {
    uint32_t max_n = 0;
    for (uint32_t j = 0; j < a.count; ++j) max_n = std::max(max_n, a.b[j].n);
    if (!max_n) return;
    if (ix.words == 1) {
        static const bool old_search = [] { const char* e = getenv("SMGX_SEARCH_V1"); return e && e[0] == '1'; }();
        const size_t smem2 = (size_t)std::max<uint32_t>(a.max_blocks, 1) * 8 * 8;
        if (old_search || smem2 > 160 * 1024 || !a.recs) event_search_thread_kernel<<<dim3((max_n + 127) / 128, a.count), 128, 0, stream>>>(ix, fleet, a);
        else {
            // requests per CTA: the fewest of 128 / 160 / 192 / 256 whose grid is still ONE wave of resident CTAs (4 per SM) — fewer requests per
            // CTA are fewer queued drains per warp, i.e. fewer rounds of dependent round trips in phase B; a second wave would cost more than that
            static const int rpc_env = [] { const char* e = getenv("SMGX_SEARCH_RPC"); return e ? atoi(e) : 0; }();   // force one of them
            int rpc = 256;
            for (int c : {128, 160, 192, 256})
                if ((uint64_t)((max_n + c - 1) / c) * a.count <= (uint64_t)sm_count * 4) { rpc = c; break; }
            if (rpc_env == 128 || rpc_env == 160 || rpc_env == 192 || rpc_env == 256) rpc = rpc_env;
            static const bool pdl = [] { const char* e = getenv("SMGX_PDL"); return !(e && e[0] == '0'); }();
            auto go = [&](auto kernel, int c) {
                if (smem2 > 32 * 1024) SMGX_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
                cudaLaunchConfig_t cfg = {};
                cfg.gridDim = dim3((max_n + c - 1) / c, a.count); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem2; cfg.stream = stream;
                cudaLaunchAttribute at[1];
                at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
                at[0].val.programmaticStreamSerializationAllowed = 1;   // may start while the preceding kernel of the stream (the hash kernel) drains
                cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
                SMGX_CUDA(cudaLaunchKernelEx(&cfg, kernel, ix, fleet, a));
            };
            if (rpc == 128) go(event_search2_kernel<128>, 128);
            else if (rpc == 160) go(event_search2_kernel<160>, 160);
            else if (rpc == 192) go(event_search2_kernel<192>, 192);
            else go(event_search2_kernel<256>, 256);
        }
    } else {
        size_t per_warp = (size_t)std::max<uint32_t>(a.max_blocks, 1) * 8;
        int wpc = 8;
        while (wpc > 1 && per_warp * wpc > 96 * 1024) wpc >>= 1;
        size_t smem = per_warp * wpc;
        if (smem > 200 * 1024) throw Error(SMGX_INVALID_ARGUMENT, "request too long for the per-warp scratch (max_tokens_per_request)");
        unsigned gx = std::min<unsigned>((max_n + wpc - 1) / wpc, (unsigned)sm_count * 16);
        if (smem > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(event_search_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        event_search_warp_kernel<<<dim3(std::max(1u, gx), a.count), wpc * 32, smem, stream>>>(ix, fleet, a);
    }
    SMGX_CUDA(cudaGetLastError());
    ++*launches;
}

// the one-launch path: ≤ 64 interned workers, counters and records present, phase C's shared-memory rows small enough to leave 4 CTAs per SM
static bool launch_event_hs(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, uint32_t max_n, cudaStream_t stream) {
    if (event_path() != 2 || ix.words != 1 || !a.group_count || !a.recs || !a.hashes || !a.block_size || a.ready) return false;
    const size_t smem = (size_t)std::max<uint32_t>(a.max_blocks, 1) * 8 * 8;
    if (smem > 40 * 1024 || (max_n + 255) / 256 > a.group_stride) return false;
    constexpr int UNR = 2;
    const uint64_t slots = (uint64_t)max_n * a.max_blocks;
    const uint64_t gx = (slots + 256 * UNR - 1) / (256 * UNR);
    if (gx == 0 || gx > 0x7FFFFFFFull) return false;
    if (a.block_size == 16) event_hs_kernel<16, UNR><<<dim3((unsigned)gx, a.count), 256, smem, stream>>>(ix, fleet, a);
    else event_hs_kernel<0, UNR><<<dim3((unsigned)gx, a.count), 256, smem, stream>>>(ix, fleet, a);
    SMGX_CUDA(cudaGetLastError());
    return true;
}

// the persistent streaming path: ≤ 64 interned workers, block size 16, ≤ 32 blocks per request (one request slot ≤ 2 KB of a 16 KB stage)
static bool launch_event_stream(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream) {
    if (event_path() != 3 || ix.words != 1 || !a.recs || !a.hashes || a.block_size != 16 || a.ready || a.max_blocks < 1 || a.max_blocks > 32) return false;
    const uint32_t R = (uint32_t)kStConsumers / a.max_blocks;
    uint64_t n_tiles = 0;
    for (uint32_t j = 0; j < a.count; ++j) n_tiles += (a.b[j].n + R - 1) / R;
    if (n_tiles == 0 || n_tiles > 0xFFFFFFFFull) return false;
    const size_t smem = (size_t)kStStages * kStStageBytes + (size_t)a.max_blocks * 7 * 8 + 2 * kStStages * 8;
    static int per_sm = -1;
    if (per_sm < 0) {
        SMGX_CUDA(cudaFuncSetAttribute(event_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kStStages * kStStageBytes + 32 * 7 * 8 + 2 * kStStages * 8)));
        int occ = 0;
        SMGX_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, event_stream_kernel, 256, kStStages * kStStageBytes + 32 * 7 * 8 + 2 * kStStages * 8));
        per_sm = std::max(occ, 1);
    }
    const unsigned grid = (unsigned)std::min<uint64_t>(n_tiles, (uint64_t)per_sm * sm_count);
    event_stream_kernel<<<grid, 256, smem, stream>>>(ix, fleet, a, (uint32_t)n_tiles);
    SMGX_CUDA(cudaGetLastError());
    return true;
}

void launch_event_select(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, int sm_count, cudaStream_t stream, uint64_t* launches) {
    if (a.count == 0) return;
    uint32_t max_n = 0;
    for (uint32_t j = 0; j < a.count; ++j) max_n = std::max(max_n, a.b[j].n);
    if (max_n == 0) return;
    if (event_launch_is_split(a)) {
        if (launch_event_stream(ix, fleet, a, sm_count, stream)) { ++*launches; return; }
        if (launch_event_hs(ix, fleet, a, max_n, stream)) { ++*launches; return; }
        launch_event_hash(a, sm_count, stream, launches);
        launch_event_search(ix, fleet, a, sm_count, stream, launches);
        return;
    }
    {
        const bool w1 = ix.words == 1;
        // one thread per request, rare shapes queued for event_slow_kernel (see event_lane_kernel)
        if (!needs_fused_kernel(a) && event_lane_selected() && w1 && a.block_size == 16 && a.slow_queue && a.max_blocks * 8 * 8 <= 200 * 1024) {
            bool plain = true;
            for (uint32_t j = 0; j < a.count; ++j) plain = plain && a.b[j].cand == nullptr;
            if (plain) {
                *launches += launch_lane(ix, fleet, a, sm_count, stream, a.slow_queue);
                return;
            }
        }
        const int tile = needs_fused_kernel(a) ? 0 : fused_tile();
        // the tiled kernel: one warp per TILE requests (see event_tile_kernel); needs uniform single-jump requests and enough tiles to fill the GPU
        if (tile && w1 && a.block_size == 16 && a.max_blocks <= 32 && ix.jump + 1 >= a.max_blocks && a.uniform_n && !a.b[0].cand &&
            (long long)a.total >= (g_tile_min_total.load(std::memory_order_relaxed) >= 0 ? g_tile_min_total.load(std::memory_order_relaxed) : (long long)tile * 4 * sm_count)) {
            bool plain = true;
            for (uint32_t j = 0; j < a.count; ++j) plain = plain && a.b[j].cand == nullptr;
            if (plain) {
                if (tile == 8) launch_tile<8>(ix, fleet, a, sm_count, stream);
                else if (tile == 32) launch_tile<32>(ix, fleet, a, sm_count, stream);
                else launch_tile<16>(ix, fleet, a, sm_count, stream);
                SMGX_CUDA(cudaGetLastError());
                ++*launches;
                return;
            }
        }
        if (a.block_size == 16) { if (w1) launch_fused<true, 16>(ix, fleet, a, sm_count, stream); else launch_fused<false, 16>(ix, fleet, a, sm_count, stream); }
        else { if (w1) launch_fused<true, 0>(ix, fleet, a, sm_count, stream); else launch_fused<false, 0>(ix, fleet, a, sm_count, stream); }
        SMGX_CUDA(cudaGetLastError());
        ++*launches;
    }
}

namespace {
// ---- load-feedback mode, phase 2: the request STREAM with the router's WorkerLoadGuard --------------------------------------------
// In the reference every request is routed by its own select_worker call and the router bumps the chosen worker's load() right after
// (routers/http/router.rs:319-321 → worker.rs:1067-1070), so request i+1 sees request i's increment: min-load picks spread over the
// fleet (water-filling), overlap ties re-read the running loads and the f32 imbalance gate is re-evaluated per request.  One warp walks
// the a.total requests in order.  Everything that does not depend on loads was done by the fused kernel (per request: the eligible
// workers tied on the best overlap score).  Running state: loads per slice entry in shared memory, global min / max over ALL workers
// (cache_aware.rs:662-666) with the number of workers at the minimum — a +1 bump changes them in O(1) except when the last worker leaves
// the minimum — and the first healthy argmin, rescanned by the warp only after it was itself picked.
__device__ __forceinline__ uint64_t warp_min_u64(uint64_t v) {
#pragma unroll
    for (int d = 16; d; d >>= 1) { uint64_t o = shfl64_xor(v, d); v = o < v ? o : v; }
    return v;
}
__global__ void __launch_bounds__(32) feedback_resolve_kernel(const __grid_constant__ EventIndexView v, FleetView f, const __grid_constant__ MultiArgs a,
                                                              const uint64_t* __restrict__ loads0, const uint8_t* __restrict__ flags, uint32_t n_slice,
                                                              uint64_t abs_thr, float rel_thr, uint64_t* loads_out) {
    extern __shared__ uint64_t s_L[];   // [n_slice]
    const int lane = threadIdx.x;
    const uint32_t n_healthy = f.derived->n_healthy;
    for (uint32_t i = lane; i < n_slice; i += 32) s_L[i] = loads0[i];
    __syncwarp();
    uint64_t gmin = f.derived->min_load, gmax = f.derived->max_load, hmin = f.derived->min_healthy_load;
    int32_t hidx = f.derived->min_load_idx;
    auto count_at = [&](uint64_t val) { uint32_t c = 0; for (uint32_t i = lane; i < n_slice; i += 32) c += s_L[i] == val; return __reduce_add_sync(FULL, c); };
    uint32_t cnt_gmin = n_slice ? count_at(gmin) : 0;
    auto rescan_healthy = [&]() {   // first argmin load over healthy (min_by_key → FIRST minimum)
        uint64_t m = ~0ULL;
        for (uint32_t i = lane; i < n_slice; i += 32) if ((flags[i] & 3) == 3 && s_L[i] < m) m = s_L[i];
        m = warp_min_u64(m);
        uint32_t first = 0xFFFFFFFFu;
        for (uint32_t i = lane; i < n_slice; i += 32) if ((flags[i] & 3) == 3 && s_L[i] == m) { first = i; break; }
        first = __reduce_min_sync(FULL, first);
        hmin = m; hidx = (int32_t)first;
    };
    uint32_t g = 0;
    for (uint32_t j = 0; j < a.count; ++j) {
        const BatchDesc& b = a.b[j];
        for (uint32_t r = 0; r < b.n; ++r, ++g) {
            int32_t out = -1;
            uint32_t branch = SMGX_BR_NO_HEALTHY, matched = 0;
            const uint32_t score = a.fb_scores[g];
            if (n_healthy == 0) continue;               // the fused kernel already wrote None for these
            if (score == 0xFFFFFFFFu) { branch = 255; }
            else {
                const bool imbalanced = (gmax - gmin) > abs_thr && __ull2float_rn(gmax) > __fmul_rn(__ull2float_rn(gmin), rel_thr);
                if (imbalanced) { out = hidx; branch = SMGX_BR_IMBALANCED_MIN_LOAD; }
                else {
                    Cand c{false, 0, 0, -1};
                    for (uint32_t w = 0; w < v.words; ++w) {
                        uint64_t bits = a.fb_winsets[(size_t)g * v.words + w];
                        while (bits) {
                            const uint32_t id = w * 64 + (uint32_t)(__ffsll((long long)bits) - 1);
                            bits &= bits - 1;
                            const int32_t sl = f.slice_of_id[id];
                            if (sl >= 0) c.consider(sl, s_L[sl], v.tree_sizes[id]);
                        }
                    }
                    if (c.have) { out = c.sl; branch = SMGX_BR_EVENT_OVERLAP; matched = score; }
                    else { out = hidx; branch = SMGX_BR_EVENT_MIN_LOAD; }
                }
            }
            if (lane == 0) {
                const uint32_t off = b.offsets[r];
                write_pick(b, r, out, branch, matched, b.offsets[r + 1] - off);
            }
            if (out >= 0) {   // WorkerLoadGuard::new → increment_load()
                const uint64_t old = s_L[out];
                __syncwarp();
                if (lane == 0) s_L[out] = old + 1;
                __syncwarp();
                if (old + 1 > gmax) gmax = old + 1;
                if (old == gmin && --cnt_gmin == 0) { gmin = old + 1; cnt_gmin = count_at(gmin); }
                if (out == hidx) rescan_healthy();
            }
        }
    }
    if (loads_out) for (uint32_t i = lane; i < n_slice; i += 32) loads_out[i] = s_L[i];
}
}  // namespace

void launch_feedback_resolve(const EventIndexView& ix, const FleetView& fleet, const MultiArgs& a, const uint64_t* d_loads, const uint8_t* d_flags,
                             uint32_t n_slice, uint64_t abs_threshold, float rel_threshold, uint64_t* d_loads_out, cudaStream_t stream) {
    const size_t smem = (size_t)std::max<uint32_t>(n_slice, 1) * 8;
    if (smem > 200 * 1024) throw Error(SMGX_INVALID_ARGUMENT, "fleet too large for the load-feedback pass");
    if (smem > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(feedback_resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    feedback_resolve_kernel<<<1, 32, smem, stream>>>(ix, fleet, a, d_loads, d_flags, n_slice, abs_threshold, rel_threshold, d_loads_out);
    SMGX_CUDA(cudaGetLastError());
}

void launch_find_matches(const EventIndexView& ix, const uint64_t* d_hashes, uint32_t n, bool early_exit, uint32_t* d_scores,
                         cudaStream_t stream) {
    size_t smem = (size_t)std::max<uint32_t>(n, 1) * 8;
    if (smem > 200 * 1024) throw Error(SMGX_INVALID_ARGUMENT, "too many content hashes for one find_matches call");
    auto k = ix.words == 1 ? find_matches_kernel<true> : find_matches_kernel<false>;
    if (smem > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<1, 32, smem, stream>>>(ix, d_hashes, n, early_exit ? 1 : 0, d_scores);
    SMGX_CUDA(cudaGetLastError());
}

void launch_content_hashes(const uint32_t* d_tokens, uint32_t n_tokens, uint32_t block_size, uint64_t* d_out, cudaStream_t stream) {
    uint32_t nb = block_size ? n_tokens / block_size : 0;
    if (!nb) return;
    content_hashes_kernel<<<(nb + 127) / 128, 128, 0, stream>>>(d_tokens, n_tokens, block_size, d_out);
    SMGX_CUDA(cudaGetLastError());
}

namespace {
// Merge step of the worker-id-sharded pick: one thread per request walks the shards in rank order (= global slice order),
// keeping max_by_key((score, Reverse(load), Reverse(tree_size))) with LAST max — the same comparison score_overlap makes over
// the whole fleet (cache_aware.rs:806-818); the prologue (healthy count, min/max load, f32 imbalance gate, first min load) is
// re-derived from the shards' summaries.
// `flags` non-null (peer-memory exchange): cands / fleets are this rank's gather buffer, written by the peers over NVLink; the CTA
// first waits until every peer's flag has reached `seq` (acquire at system scope), and the data is read past L1 (ld.cg) because
// the same buffer held other values two steps ago.  fleet_stride: bytes between two shards' summaries.
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__global__ void __launch_bounds__(256) shard_reduce_kernel(const smgx_shard_candidate* cands, const uint8_t* fleets, uint32_t fleet_stride,
                                                           const uint32_t* __restrict__ gbase, uint32_t world, uint32_t n, uint32_t cand_stride,
                                                           uint64_t abs_thr, float rel_thr, int32_t* __restrict__ out_idx,
                                                           smgx_decision_info* __restrict__ out_info, const uint64_t* flags, uint64_t seq,
                                                           uint32_t* err_flag) {
    if (flags) {
        if (threadIdx.x < world) {
            const long long t0 = clock64();
            while (ld_acquire_sys(flags + threadIdx.x) < seq) {
                if (clock64() - t0 > 40000000000LL) { if (err_flag) atomicExch(err_flag, 2u); break; }   // ≈20 s: a peer never arrived
                __nanosleep(200);
            }
        }
        __syncthreads();
    }
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    uint64_t mn = ~0ULL, mx = 0, hl = ~0ULL;
    uint32_t n_healthy = 0;
    int32_t min_idx = -1;
    for (uint32_t g = 0; g < world; ++g) {
        smgx_shard_fleet f;
        {
            const uint64_t* fp = reinterpret_cast<const uint64_t*>(fleets + (size_t)g * fleet_stride);
            uint64_t w[5];
#pragma unroll
            for (int i = 0; i < 5; ++i) w[i] = __ldcg(fp + i);
            memcpy(&f, w, sizeof(f));
        }
        mn = f.min_load < mn ? f.min_load : mn;
        mx = f.max_load > mx ? f.max_load : mx;
        n_healthy += f.n_healthy;
        if (f.n_healthy && f.min_healthy_load < hl) { hl = f.min_healthy_load; min_idx = (int32_t)(gbase[g] + (uint32_t)f.min_load_idx); }   // strict <: FIRST min
    }
    if (mn == ~0ULL) mn = 0;   // no worker on any shard (or every load at UINT64_MAX): cache_aware.rs:666
    int32_t out = -1;
    uint32_t branch = SMGX_BR_NO_HEALTHY, matched = 0;
    if (n_healthy) {
        const bool imbalanced = (mx - mn) > abs_thr && __ull2float_rn(mx) > __fmul_rn(__ull2float_rn(mn), rel_thr);
        if (imbalanced) { out = min_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD; }
        else {
            bool have = false;
            uint32_t bs = 0; uint64_t bl = 0, bt = 0; int32_t bi = -1;
            for (uint32_t g = 0; g < world; ++g) {
                smgx_shard_candidate c;
                {
                    const uint64_t* cp = reinterpret_cast<const uint64_t*>(cands + (size_t)g * cand_stride + r);
                    uint64_t w[3];
#pragma unroll
                    for (int i = 0; i < 3; ++i) w[i] = __ldcg(cp + i);
                    memcpy(&c, w, sizeof(c));
                }
                if (c.score == 0 || c.local_idx == 0xFFFFFFFFu) continue;
                const bool ge = !have || c.score > bs || (c.score == bs && (c.load < bl || (c.load == bl && c.tree_size <= bt)));   // >= : LAST max
                if (ge) { have = true; bs = c.score; bl = c.load; bt = c.tree_size; bi = (int32_t)(gbase[g] + c.local_idx); }
            }
            if (have) { out = bi; branch = SMGX_BR_EVENT_OVERLAP; matched = bs; }
            else { out = min_idx; branch = SMGX_BR_EVENT_MIN_LOAD; }
        }
    }
    out_idx[r] = out;
    if (out_info) {
        smgx_decision_info di;
        di.matched = matched; di.input = 0; di.branch = (uint8_t)branch;
        di.nodes = 0; di.reserved[0] = di.reserved[1] = 0;
        out_info[r] = di;
    }
}

// Push this shard's candidates + summary into EVERY rank's gather buffer (slot `rank`) over peer memory, then raise this rank's
// flag there: the CTAs write their share, fence at system scope and count themselves in; the last one to arrive publishes `seq`.
__global__ void __launch_bounds__(256) shard_push_kernel(const uint64_t* __restrict__ cand_words, uint32_t n_words, const uint64_t* __restrict__ fleet_words,
                                                         uint8_t* const* __restrict__ peer_parity_base, uint32_t world, uint32_t rank, size_t cand_off,
                                                         size_t cand_slot_bytes, size_t fleet_off, uint32_t fleet_stride, size_t flag_off, uint64_t seq,
                                                         uint32_t* __restrict__ arrive) {
    const uint32_t q = blockIdx.y;
    uint8_t* base = peer_parity_base[q];
    uint64_t* dst = reinterpret_cast<uint64_t*>(base + cand_off + (size_t)rank * cand_slot_bytes);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += gridDim.x * blockDim.x) dst[i] = cand_words[i];
    if (blockIdx.x == 0 && threadIdx.x < 5) reinterpret_cast<uint64_t*>(base + fleet_off + (size_t)rank * fleet_stride)[threadIdx.x] = fleet_words[threadIdx.x];
    __threadfence_system();
    __syncthreads();
    __shared__ bool last;
    if (threadIdx.x == 0) last = atomicAdd(arrive, 1u) == gridDim.x * gridDim.y - 1;
    __syncthreads();
    if (last) {
        __threadfence_system();
        if (threadIdx.x < world) {
            uint64_t* f = reinterpret_cast<uint64_t*>(peer_parity_base[threadIdx.x] + flag_off) + rank;
            asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(f), "l"(seq) : "memory");
        }
        if (threadIdx.x == 0) *arrive = 0;
    }
}
}  // namespace

void launch_shard_push(const smgx_shard_candidate* d_cand, uint32_t n, const smgx_shard_fleet* d_fleet, uint8_t* const* d_peer_parity_base, uint32_t world,
                       uint32_t rank, size_t cand_off, size_t cand_slot_bytes, size_t fleet_off, uint32_t fleet_stride, size_t flag_off, uint64_t seq,
                       uint32_t* d_arrive, cudaStream_t stream) {
    const uint32_t n_words = n * 3;   // 24 B per candidate
    dim3 grid(std::max<uint32_t>(1, std::min<uint32_t>((n_words + 255) / 256, 64)), world);
    shard_push_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint64_t*>(d_cand), n_words, reinterpret_cast<const uint64_t*>(d_fleet),
                                               d_peer_parity_base, world, rank, cand_off, cand_slot_bytes, fleet_off, fleet_stride, flag_off, seq, d_arrive);
    SMGX_CUDA(cudaGetLastError());
}

void launch_shard_reduce(const smgx_shard_candidate* d_cands, const smgx_shard_fleet* d_fleets, const uint32_t* d_global_base, uint32_t world,
                         uint32_t n, uint64_t abs_threshold, float rel_threshold, int32_t* d_out_idx, smgx_decision_info* d_out_info,
                         cudaStream_t stream) {
    if (!n) return;
    shard_reduce_kernel<<<(n + 255) / 256, 256, 0, stream>>>(d_cands, reinterpret_cast<const uint8_t*>(d_fleets), (uint32_t)sizeof(smgx_shard_fleet),
                                                             d_global_base, world, n, n, abs_threshold, rel_threshold, d_out_idx, d_out_info, nullptr, 0, nullptr);
    SMGX_CUDA(cudaGetLastError());
}
void launch_shard_reduce_wait(const uint8_t* d_parity_base, size_t cand_off, uint32_t cand_stride, size_t fleet_off, uint32_t fleet_stride, size_t flag_off,
                              uint64_t seq, const uint32_t* d_global_base, uint32_t world, uint32_t n, uint64_t abs_threshold, float rel_threshold,
                              int32_t* d_out_idx, smgx_decision_info* d_out_info, uint32_t* d_err, cudaStream_t stream) {
    shard_reduce_kernel<<<std::max<uint32_t>(1, (n + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const smgx_shard_candidate*>(d_parity_base + cand_off), d_parity_base + fleet_off, fleet_stride, d_global_base, world, n, cand_stride,
        abs_threshold, rel_threshold, d_out_idx, d_out_info, reinterpret_cast<const uint64_t*>(d_parity_base + flag_off), seq, d_err);
    SMGX_CUDA(cudaGetLastError());
}

void launch_content_hashes_ragged(const uint32_t* d_tokens, const uint32_t* d_offs, uint32_t n_blocks, uint64_t* d_out, cudaStream_t stream) {
    if (!n_blocks) return;
    content_hashes_ragged_kernel<<<(n_blocks + 127) / 128, 128, 0, stream>>>(d_tokens, d_offs, n_blocks, d_out);
    SMGX_CUDA(cudaGetLastError());
}

namespace {
__global__ void hold_kernel(unsigned long long ns) {
    unsigned long long t0, t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    do { __nanosleep(200); asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); } while (t - t0 < ns);
}
}  // namespace
// Keeps `stream` busy for ~`us` microseconds: bench.py enqueues a whole timed region behind it, so the CUDA events that bracket the region
// see GPU execution only, not the host's launch latency.
void launch_hold(uint32_t us, cudaStream_t stream) {
    hold_kernel<<<1, 1, 0, stream>>>((unsigned long long)us * 1000ull);
    SMGX_CUDA(cudaGetLastError());
}

void launch_fill(uint32_t* d, uint32_t value, size_t n_words, cudaStream_t stream) {
    if (!n_words) return;
    unsigned grid = (unsigned)std::min<size_t>((n_words + 255) / 256, (size_t)current_sm_count() * 8);
    fill_kernel<<<grid, 256, 0, stream>>>(d, value, n_words);
    SMGX_CUDA(cudaGetLastError());
}

}  // namespace smgx
