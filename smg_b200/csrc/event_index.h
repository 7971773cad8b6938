// GPU-resident positional KV index: host-side writer + device mirror.
//
// Product counterpart of kv_index::PositionalIndexer (crates/kv_index/src/event_tree.rs:257-271).  The reference
// keeps `DashMap<(position, ContentHash), SeqEntry>` whose values own FxHashSet<u32> worker sets; here the index
// is ONE open-addressed table of 32-byte slots in HBM (one sector per probe) with worker sets as bitsets:
//
//   Slot   { u64 content_hash; u32 position; u32 state; u32 run; u32 pad; u64 payload }          32 B, 32 B-aligned
//          state SINGLE: SeqEntry::Single(prefix_hash, set)   payload = the bitset itself when the fleet has ≤ 64
//                                                              interned workers, else a row number into `rows`
//          state MULTI : SeqEntry::Multi(map)                  payload = head of a linked list in `multi`
//          run: the entry's record in `runs` (kNil for none).  A Single entry's prefix_hash is host-only (`prefix_`, parallel
//          to the slots): no kernel reads it
//   runs   [n_runs] RunRec { u64 content_hash; u32 position; u32 state; u64 payload; u64 pad }  32 B, append-only
//          each apply_stored call reserves one run of consecutive records, one per block in position order, so that within a
//          run record index = anchor + position.  A block that creates its key fills its record and the slot's `run` points at
//          it; a block whose key already exists leaves its record dead (state EMPTY).  A live record (SINGLE / MULTI) exists only
//          for a key that is live in the slots, with the slot's state and payload: keys are unique, so a key match in ANY live
//          record is that entry, wherever the record lies.  A drain reads the records of a stored sequence's positions as one
//          contiguous range from the anchor of its position-0 slot, in the same round trip as their tokens, where the slots
//          are one cold HBM read each behind a tag round trip.  Compacted whole runs at a time (runs with no live record are
//          dropped, records never move inside a run) at a rebuild, or when dead records outnumber live entries and the arena has
//          doubled since the last compaction
//   rows   [n_rows][words] u64                                 worker bitsets (words = ceil(workers/64) → pow2, ≤ 32)
//   multi  { u64 prefix_hash; u64 payload; u32 next; ... }     32 B nodes; one per distinct prefix hash
//   tree_sizes[worker] u64                                     event_tree.rs:264
//   tags   [capacity] u8                                       one byte per slot, derived on the device from the slots: 0 empty,
//                                                              1 tombstone, tag_of(pos, content) ∈ 2..255 for a live key
//
// The slots are far larger than L2 (32 B each at ≤ 25 % load: 128 MiB for 1 M entries, most 128 B lines holding a live slot), so a
// probe that reads a slot only to find a different key or an empty one is an HBM round trip that carries one bit.  The tag array is
// 1 B per slot (4 MiB at 4 M slots) and stays in L2: a collision chain is walked in the tags, and a slot is read only where the tag
// matches, then its full key is compared.
//
// Writers (apply_stored / apply_removed / apply_cleared / remove_worker, event_tree.rs:305-435) run on the host
// against an identical host mirror and record dirty slots; flush() pushes them to the device with one scatter
// kernel (or a bulk copy after a rebuild) in stream order before the next query batch.  Queries never touch the
// host copy.
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.h"

namespace smgx {

enum : uint32_t { SLOT_EMPTY = 0, SLOT_SINGLE = 1, SLOT_MULTI = 2, SLOT_TOMB = 3 };
constexpr uint32_t kNil = 0xFFFFFFFFu;
constexpr uint32_t kMaxWords = 32;  // 2048 workers per device shard (reference MAX_WORKERS, event_tree.rs:48)

struct alignas(32) Slot {
    uint64_t content;
    uint32_t pos;
    uint32_t state;
    uint32_t run;
    uint32_t pad;
    uint64_t payload;
};
struct alignas(32) RunRec {
    uint64_t content;
    uint32_t pos;
    uint32_t state;   // the slot's state while the key is live in it; SLOT_EMPTY for a dead record
    uint64_t payload;
    uint64_t pad;
};
struct alignas(32) MultiNode {
    uint64_t prefix;
    uint64_t payload;
    uint32_t next;
    uint32_t pad0;
    uint64_t pad1;
};
static_assert(sizeof(Slot) == 32 && sizeof(MultiNode) == 32 && sizeof(RunRec) == 32, "32-byte records");

// What the kernels see.
struct EventIndexView {
    const Slot* slots;
    const uint64_t* rows;
    const MultiNode* multi;
    const uint64_t* tree_sizes;
    const uint8_t* tags; // one tag per slot (see above)
    const RunRec* runs;  // the run arena (see above)
    uint32_t n_runs;     // records in it
    uint32_t mask;       // capacity - 1
    uint32_t words;      // u64 words per worker bitset
    uint32_t n_workers;  // interned workers
    uint32_t jump;       // jump_size (event_tree.rs:270)
};

__host__ __device__ inline uint64_t key_hash(uint32_t pos, uint64_t content) {
    return (content ^ ((uint64_t)pos * 0x9E3779B97F4A7C15ULL)) * 0xD6E8FEB86659FD93ULL;
}
// home slot: the high half of the key hash (masked to the capacity)
__host__ __device__ inline uint32_t slot_hash(uint32_t pos, uint64_t content) { return (uint32_t)(key_hash(pos, content) >> 32); }
// tag of a live key, 2..255: bits 16..31 of the key hash, which no capacity's home slot uses, reduced to 254 values
enum : uint8_t { TAG_EMPTY = 0, TAG_TOMB = 1 };
__host__ __device__ inline uint8_t tag_of(uint32_t pos, uint64_t content) {
    return (uint8_t)(2u + ((((uint32_t)key_hash(pos, content) >> 16) * 254u) >> 16));
}
__host__ __device__ inline uint8_t slot_tag(uint32_t state, uint32_t pos, uint64_t content) {
    return state == SLOT_EMPTY ? (uint8_t)TAG_EMPTY : state == SLOT_TOMB ? (uint8_t)TAG_TOMB : tag_of(pos, content);
}

struct BlockRec { uint32_t pos; uint64_t content; uint64_t prefix; };

class EventIndex {
public:
    explicit EventIndex(uint32_t jump_size);
    ~EventIndex();
    EventIndex(const EventIndex&) = delete;

    // ---- writer side (host) ----
    uint32_t intern_worker(const std::string& url);                       // event_tree.rs:509-525
    int64_t worker_id(const std::string& url) const;                      // :294
    smgx_status apply_stored(uint32_t wid, const uint64_t* seq, const uint64_t* content, uint32_t n, const uint64_t* parent);
    void apply_removed(uint32_t wid, const uint64_t* seq, uint32_t n);
    void apply_cleared(uint32_t wid);
    void remove_worker(uint32_t wid);
    uint64_t current_size() const;                                        // :438-444
    uint64_t entry_count() const { return live_; }
    // slots in state MULTI: while there is none, no lookup can need a rolling prefix hash
    uint64_t multi_count() const { return multi_slots_; }
    uint32_t n_workers() const { return (uint32_t)tree_sizes_.size(); }
    uint32_t jump() const { return jump_; }
    uint64_t workers_version() const { return workers_version_; }
    uint32_t words() const { return words_; }
    uint64_t tree_size(uint32_t wid) const { return tree_sizes_[wid]; }

    // ---- device side ----
    // Push pending writes to the device in `stream` order and return the view for kernels.
    EventIndexView flush(cudaStream_t stream, uint64_t* launches);
    bool device_enabled = true;
    bool pending() const {
        return full_dirty_ || tree_dirty_ || !dirty_slots_.empty() || !dirty_multi_.empty() || !dirty_rows_.empty() || !dirty_runs_.empty();
    }

private:
    // bitset helpers on the HOST mirror
    uint64_t* set_words(uint64_t& payload);
    uint64_t new_set(uint32_t wid);
    void free_set(uint64_t payload);
    bool set_empty(uint64_t& payload);
    void mark_set_dirty(uint64_t payload);

    int64_t find_slot(uint32_t pos, uint64_t content) const;
    uint32_t insert_slot(uint32_t pos, uint64_t content);
    void insert_entry(uint32_t pos, uint64_t content, uint64_t prefix, uint32_t wid, uint32_t i);
    void drop_entry(const BlockRec& r, uint32_t wid);
    uint32_t new_multi(uint64_t prefix, uint64_t payload, uint32_t next);
    void rebuild(uint32_t new_capacity, uint32_t new_words);
    void compact_runs();
    // every write to a slot's state or payload goes through here: it rewrites the slot's record as well
    void mark_slot(uint32_t i) {
        if (!full_dirty_) dirty_slots_.push_back(i);
        const Slot& s = slots_[i];
        if (s.run == kNil) return;
        const bool live = s.state == SLOT_SINGLE || s.state == SLOT_MULTI;
        runs_[s.run] = RunRec{s.content, s.pos, live ? s.state : (uint32_t)SLOT_EMPTY, live ? s.payload : 0, 0};
        if (!full_dirty_) dirty_runs_.push_back(s.run);
    }
    void mark_multi(uint32_t i) { if (!full_dirty_) dirty_multi_.push_back(i); }
    void mark_row(uint32_t i) { if (!full_dirty_) dirty_rows_.push_back(i); }

    uint32_t jump_;
    uint32_t words_ = 1;
    std::vector<Slot> slots_;
    std::vector<uint64_t> prefix_;        // a Single entry's prefix hash, per slot (host only)
    std::vector<RunRec> runs_;
    std::vector<uint32_t> run_starts_;    // first record of each run, ascending
    size_t runs_kept_ = 0;                // records left by the last compaction
    uint32_t mask_ = 0;
    uint64_t live_ = 0, tombs_ = 0, multi_slots_ = 0;
    std::vector<uint64_t> rows_;
    std::vector<uint32_t> free_rows_;
    std::vector<MultiNode> multi_;
    std::vector<uint32_t> free_multi_;
    std::vector<uint64_t> tree_sizes_;
    std::vector<std::unordered_map<uint64_t, BlockRec>> worker_blocks_;  // WorkerBlockMap per worker (event_tree.rs:246)
    std::unordered_map<std::string, uint32_t> worker_to_id_;
    uint64_t workers_version_ = 0;

    // device mirror
    DevBuf d_slots_, d_rows_, d_multi_, d_tree_, d_tags_, d_runs_;
    PinBuf stage_;
    DevBuf d_stage_;
    cudaEvent_t stage_done_ = nullptr;
    bool stage_pending_ = false;
    bool full_dirty_ = true;
    bool tree_dirty_ = true;
    std::vector<uint32_t> dirty_slots_, dirty_multi_, dirty_rows_, dirty_runs_;
};

}  // namespace smgx
