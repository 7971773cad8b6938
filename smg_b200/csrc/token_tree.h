// K2a — approximate token tree: host-authoritative radix tree + device mirror for the match/decide kernel.
//
// Product counterpart of kv_index::TokenTree (crates/kv_index/src/token_tree.rs): page-aligned (16-token) multi-tenant
// radix tree.  Mutations (insert_tokens :401-609, touch_tenant :291-314, eviction :798-1024) run on the host in request
// order — every routed request inserts, so the tree changes after every decision — while the longest-prefix match of a
// whole conflict-free segment of requests (match_prefix_with_counts :615-740) and the pick run on the GPU against the
// mirror:
//   tokens   [n] u32          append-only arena of edge labels; a split re-slices, it never copies
//   slots    [cap] 32 B       open-addressed { u64 key; u32 parent; u32 child; u64 label_off; u32 label_len; i32 any_tenant },
//                             key = hash(parent, 16-token page key); the child's header is embedded so a probe hit needs no
//                             second dependent read.  any_tenant = get_any_tenant() (:268-284), evaluated on the host whenever
//                             the node's tenants / last_tenant change (−1 = no tenants)
// Device-side insertion is the §8(f) "next" item; DESIGN.md explains the segment scheme that keeps sequential semantics.
#pragma once
#include <cstdint>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.h"

namespace smgx {

constexpr uint32_t kPage = 16;            // token_tree.rs:44
constexpr uint32_t kNoNode = 0xFFFFFFFFu;
constexpr uint32_t kTombChild = 0xFFFFFFFEu;
constexpr uint32_t kPathCap = 32;         // matched nodes reported per request by the kernel (deeper paths are re-walked on the host)

struct alignas(16) ChildSlot { uint64_t key; uint32_t parent; uint32_t child; };  // host table entry; key 0 = empty
// device table entry: the child's header rides in the slot, so one 32 B read resolves a probe AND yields the label location
struct alignas(16) TreeSlot { uint64_t key; uint32_t parent; uint32_t child; uint64_t label_off; uint32_t label_len; int32_t any_tenant; };
static_assert(sizeof(TreeSlot) == 32, "device slot layout");

struct TokenTreeView {
    const uint32_t* tokens;
    const TreeSlot* slots;
    uint32_t child_mask;
};

// key of (parent node, first 16 tokens of the edge) — identical on host and device.  Two multilinear 32-bit hashes of the page
// (odd per-position multipliers) are summed across the warp with one redux.sync each, then mixed with the parent id.  A key
// collision is harmless: both sides still compare the page itself.
__host__ __device__ inline uint32_t page_mult1(uint32_t i) { uint32_t x = (i + 1) * 0x9E3779B9u; x ^= x >> 15; x *= 0x85EBCA6Bu; x ^= x >> 13; return x | 1u; }
__host__ __device__ inline uint32_t page_mult2(uint32_t i) { uint32_t x = (i + 17) * 0xC2B2AE35u; x ^= x >> 16; x *= 0x27D4EB2Fu; x ^= x >> 14; return x | 1u; }
__host__ __device__ inline uint64_t page_finish(uint32_t h1, uint32_t h2, uint32_t parent) {
    uint32_t a = h1 ^ (parent * 0x85EBCA6Bu + 0xC2B2AE35u);
    a ^= a >> 16; a *= 0x7FEB352Du; a ^= a >> 15; a *= 0x846CA68Bu; a ^= a >> 16;
    uint32_t b = h2 + parent * 0x27D4EB2Fu;
    b ^= b >> 15; b *= 0x2C1B3C6Du; b ^= b >> 12; b *= 0x297A2D39u; b ^= b >> 15;
    return (((uint64_t)a << 32) | b) | 1ULL;   // never 0 (0 marks an empty slot)
}
inline uint64_t page_key_host(const uint32_t* page, uint32_t parent) {
    static const struct Mults { uint32_t m1[kPage], m2[kPage]; Mults() { for (uint32_t i = 0; i < kPage; ++i) { m1[i] = page_mult1(i); m2[i] = page_mult2(i); } } } M;
    uint32_t h1 = 0, h2 = 0;
    for (uint32_t i = 0; i < kPage; ++i) { h1 += (page[i] + 1u) * M.m1[i]; h2 += (page[i] ^ 0x9E3779B9u) * M.m2[i]; }
    return page_finish(h1, h2, parent);
}

enum EvictPolicy : int { EVP_LRU = 0, EVP_LFU = 1, EVP_FIFO = 2, EVP_MRU = 3, EVP_FILO = 4, EVP_PRIORITY = 5 };

// process-wide tenant interning (token_tree.rs:160-176) — one table per policy here
struct TenantTable {
    std::vector<std::string> names;
    std::unordered_map<std::string, uint32_t> ids;
    std::vector<uint32_t> rank;   // rank[id] = position of names[id] in lexicographic order (the "any tenant" rule, DESIGN.md §3)
    uint64_t version = 0;
    uint32_t intern(const std::string& s);
    int64_t find(const std::string& s) const { auto it = ids.find(s); return it == ids.end() ? -1 : (int64_t)it->second; }
};

struct TreeMatch { int32_t tenant; uint32_t matched; uint32_t input; std::vector<uint32_t> path; std::vector<int32_t> path_tenants; };

class TokenTreeIndex {
public:
    TokenTreeIndex(TenantTable* tenants, uint64_t* global_ts, EvictPolicy policy);
    ~TokenTreeIndex();

    // ---- reference API, host side ----
    void insert_tokens(const uint32_t* toks, size_t n, uint32_t tenant);                    // :401-609
    TreeMatch match_prefix_host(const uint32_t* toks, size_t n, bool touch);                // :615-740 (host walk; used for paths deeper than kPathCap)
    void apply_match_touches(const uint32_t* path, uint32_t path_len);                      // touch_tenant on the matched nodes, in order (:685-689)
    void apply_match_touches(const uint32_t* path, const int32_t* path_tenants, uint32_t path_len);   // same, with the tenants the walk read
    void evict_tenant(uint32_t tenant, size_t max_tokens);                                  // :798-863
    void evict_tenant_by_size(size_t max_size);                                             // :1011-1024
    size_t tenant_token_size(uint32_t tenant) const;
    void clear();                                                                           // :997-1001
    size_t node_count() const { return live_nodes_; }
    void entries(std::vector<std::pair<std::vector<uint32_t>, std::vector<std::pair<uint32_t, uint64_t>>>>& out) const;  // iter_entries :1039
    int32_t any_tenant(uint32_t node) const;
    // optimistic batching (smgx.cu tree_select): nodes split since begin_chunk(), a node's label length, child lookup
    void begin_chunk() { ++chunk_epoch_; }
    bool split_in_chunk(uint32_t node) const { return nodes_[node].split_epoch == chunk_epoch_; }
    uint32_t label_len_of(uint32_t node) const { return nodes_[node].label_len; }
    bool has_child(uint32_t node, const uint32_t* page) const { return find_child(node, page) >= 0; }

    // ---- device mirror ----
    TokenTreeView flush(cudaStream_t stream, uint64_t* launches);
    bool pending() const { return full_dirty_ || !dirty_nodes_.empty() || !dirty_slots_.empty() || uploaded_tokens_ != tokens_.size(); }
    bool device_enabled = true;
    uint64_t tenants_version_seen = ~0ULL;   // any_tenant caches depend on the lexicographic ranks

    void refresh_all_any_tenant();           // after a new tenant changed the ranks

private:
    struct Node {
        uint64_t label_off = 0;
        uint32_t label_len = 0;
        uint32_t parent = kNoNode;
        std::vector<std::pair<uint32_t, uint64_t>> tenants;   // (tenant id, last access ts), unsorted, small
        int32_t last_tenant = -1;
        uint64_t hit_count = 0, creation_time = 0;
        int32_t priority = 0;
        std::vector<uint32_t> kids;                            // child node ids (for eviction / iteration)
        bool alive = true;
        uint32_t slot = kNoNode;                               // table_ index of the entry that points at this node
        uint64_t split_epoch = 0;                              // chunk in which this node was last split (or created by a split)
    };
    uint64_t next_ts() { return (*global_ts_)++; }
    uint64_t key_of(uint32_t parent, const uint32_t* page) const;
    int64_t find_child(uint32_t parent, const uint32_t* page) const;
    void table_insert(uint32_t parent, const uint32_t* page, uint32_t child);
    void table_erase(uint32_t parent, const uint32_t* page);
    void table_rebuild(uint32_t cap);
    uint32_t new_node(uint64_t off, uint32_t len, uint32_t parent, bool draw_ts);
    void free_node(uint32_t id);
    void touch(uint32_t node, uint32_t tenant);
    bool has_tenant(const Node& nd, uint32_t t) const;
    void set_tenant_ts(Node& nd, uint32_t t, uint64_t ts);
    void mark_node(uint32_t id) { if (!full_dirty_) dirty_nodes_.push_back(id); }
    void mark_slot(uint32_t i) {   // each slot at most once per flush generation: no sort / unique at flush time
        if (full_dirty_) return;
        if (slot_stamp_.size() < table_.size()) slot_stamp_.assign(table_.size(), 0);
        if (slot_stamp_[i] != flush_gen_) { slot_stamp_[i] = flush_gen_; dirty_slots_.push_back(i); }
    }
    const uint32_t* label(const Node& nd) const { return tokens_.data() + nd.label_off; }

    TenantTable* tenants_;
    uint64_t* global_ts_;
    uint64_t chunk_epoch_ = 1;
    EvictPolicy policy_;
    std::vector<Node> nodes_;            // nodes_[0] = root
    std::vector<uint32_t> free_nodes_;
    size_t live_nodes_ = 0;
    std::vector<uint32_t> tokens_;
    std::vector<ChildSlot> table_;
    uint32_t mask_ = 0;
    uint64_t table_live_ = 0, table_tombs_ = 0;
    std::vector<size_t> tenant_tokens_;                    // tenant_token_count (token_tree.rs:328), indexed by tenant id
    std::vector<uint8_t> tenant_known_;                    // … and whether the tenant has an entry at all
    std::vector<uint8_t> root_has_;                        // whether the root lists the tenant (eviction can remove it)
    std::vector<uint32_t> slot_stamp_;
    uint32_t flush_gen_ = 1;

    DevBuf d_tokens_, d_table_, d_stage_;
    TreeSlot device_slot(uint32_t i) const;
    PinBuf stage_;
    cudaEvent_t stage_done_ = nullptr;
    bool stage_pending_ = false;
    size_t uploaded_tokens_ = 0;
    bool full_dirty_ = true;
    std::vector<uint32_t> dirty_nodes_, dirty_slots_;
};

// ---- kernels (token_tree.cu) ----
struct TreeSelectArgs {
    const uint32_t* tokens;      // device, ragged
    const uint32_t* offsets;     // device, n + 1 (absolute)
    uint32_t first;              // first request of this segment
    uint32_t count;              // requests in this segment
    int32_t* out_idx;            // [n]
    smgx_decision_info* out_info;  // [n]
    uint32_t* out_path;          // [n][kPathCap]
    int32_t* out_path_tenant;    // [n][kPathCap] any-tenant each matched node had when it was read
    uint32_t* out_path_len;      // [n] (total matched nodes, may exceed kPathCap)
    int32_t* out_tenant;         // [n] any-tenant of the deepest matched node (−1 = "empty")
    float cache_threshold;
    int decide;                  // 0 = match only (TokenTree::match_prefix_with_counts API), 1 = full pick
};
struct FleetView;
void launch_tree_select(const TokenTreeView& tv, const FleetView& fleet, const int32_t* d_slice_of_tenant, const uint8_t* d_flags,
                        uint32_t n_tenants, const TreeSelectArgs& a, cudaStream_t stream);

}  // namespace smgx
