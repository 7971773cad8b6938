// GPU-resident positional KV index: host-side writer + device mirror.
//
// Product counterpart of kv_index::PositionalIndexer (crates/kv_index/src/event_tree.rs:257-271).  The reference
// keeps `DashMap<(position, ContentHash), SeqEntry>` whose values own FxHashSet<u32> worker sets; here the index
// is ONE open-addressed table of 32-byte slots in HBM (one sector per probe) with worker sets as bitsets:
//
//   Slot   { u64 content_hash; u32 position; u32 state; u64 prefix_hash; u64 payload }         32 B, 32 B-aligned
//          state SINGLE: SeqEntry::Single(prefix_hash, set)   payload = the bitset itself when the fleet has ≤ 64
//                                                              interned workers, else a row number into `rows`
//          state MULTI : SeqEntry::Multi(map)                  payload = head of a linked list in `multi`
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
    uint64_t prefix;
    uint64_t payload;
};
struct alignas(32) MultiNode {
    uint64_t prefix;
    uint64_t payload;
    uint32_t next;
    uint32_t pad0;
    uint64_t pad1;
};
static_assert(sizeof(Slot) == 32 && sizeof(MultiNode) == 32, "32-byte records");

// What the kernels see.
struct EventIndexView {
    const Slot* slots;
    const uint64_t* rows;
    const MultiNode* multi;
    const uint64_t* tree_sizes;
    const uint8_t* tags; // one tag per slot (see above)
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
    bool pending() const { return full_dirty_ || tree_dirty_ || !dirty_slots_.empty() || !dirty_multi_.empty() || !dirty_rows_.empty(); }

private:
    // bitset helpers on the HOST mirror
    uint64_t* set_words(uint64_t& payload);
    uint64_t new_set(uint32_t wid);
    void free_set(uint64_t payload);
    bool set_empty(uint64_t& payload);
    void mark_set_dirty(uint64_t payload);

    int64_t find_slot(uint32_t pos, uint64_t content) const;
    uint32_t insert_slot(uint32_t pos, uint64_t content);
    void insert_entry(uint32_t pos, uint64_t content, uint64_t prefix, uint32_t wid);
    void drop_entry(const BlockRec& r, uint32_t wid);
    uint32_t new_multi(uint64_t prefix, uint64_t payload, uint32_t next);
    void rebuild(uint32_t new_capacity, uint32_t new_words);
    void mark_slot(uint32_t i) { if (!full_dirty_) dirty_slots_.push_back(i); }
    void mark_multi(uint32_t i) { if (!full_dirty_) dirty_multi_.push_back(i); }
    void mark_row(uint32_t i) { if (!full_dirty_) dirty_rows_.push_back(i); }

    uint32_t jump_;
    uint32_t words_ = 1;
    std::vector<Slot> slots_;
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
    DevBuf d_slots_, d_rows_, d_multi_, d_tree_, d_tags_;
    PinBuf stage_;
    DevBuf d_stage_;
    cudaEvent_t stage_done_ = nullptr;
    bool stage_pending_ = false;
    bool full_dirty_ = true;
    bool tree_dirty_ = true;
    std::vector<uint32_t> dirty_slots_, dirty_multi_, dirty_rows_;
};

}  // namespace smgx
