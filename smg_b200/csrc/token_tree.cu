// K2a — approximate token tree: host tree + device mirror + the match/decide kernel.  See token_tree.h.
#include "token_tree.h"

#include <algorithm>
#include <climits>
#include <cstring>
#include <queue>

#include <cooperative_groups.h>
#include <cstdlib>

#include "kernels.h"

namespace smgx {

// =================================================================================================================
// tenant interning
// =================================================================================================================
uint32_t TenantTable::intern(const std::string& s) {
    auto it = ids.find(s);
    if (it != ids.end()) return it->second;
    uint32_t id = (uint32_t)names.size();
    names.push_back(s);
    ids[s] = id;
    std::vector<uint32_t> order(names.size());
    for (uint32_t i = 0; i < order.size(); ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return names[a] < names[b]; });
    rank.assign(names.size(), 0);
    for (uint32_t r = 0; r < order.size(); ++r) rank[order[r]] = r;
    ++version;
    return id;
}

// =================================================================================================================
// host tree
// =================================================================================================================
TokenTreeIndex::TokenTreeIndex(TenantTable* tenants, uint64_t* global_ts, EvictPolicy policy)
    : tenants_(tenants), global_ts_(global_ts), policy_(policy) {
    nodes_.emplace_back();
    nodes_[0].priority = INT_MIN;   // Node::new_root (token_tree.rs:239-254)
    table_.assign(1024, ChildSlot{0, 0, 0});
    mask_ = 1023;
}
TokenTreeIndex::~TokenTreeIndex() {
    d_tokens_.release(); d_table_.release(); d_stage_.release(); stage_.release();
    if (stage_done_) cudaEventDestroy(stage_done_);
}

uint64_t TokenTreeIndex::key_of(uint32_t parent, const uint32_t* page) const {
    return page_key_host(page, parent);
}
int64_t TokenTreeIndex::find_child(uint32_t parent, const uint32_t* page) const {
    const uint64_t h = key_of(parent, page);
    uint32_t idx = (uint32_t)(h >> 32) & mask_;
    for (;;) {
        const ChildSlot& s = table_[idx];
        if (s.key == 0) return -1;
        if (s.key == h && s.parent == parent && s.child < kTombChild &&
            memcmp(label(nodes_[s.child]), page, kPage * 4) == 0) return idx;
        idx = (idx + 1) & mask_;
    }
}
void TokenTreeIndex::table_rebuild(uint32_t cap) {
    std::vector<ChildSlot> old;
    old.swap(table_);
    table_.assign(cap, ChildSlot{0, 0, 0});
    mask_ = cap - 1;
    table_live_ = table_tombs_ = 0;
    for (const ChildSlot& s : old) {
        if (s.key == 0 || s.child >= kTombChild) continue;
        uint32_t idx = (uint32_t)(s.key >> 32) & mask_;
        while (table_[idx].key != 0) idx = (idx + 1) & mask_;
        table_[idx] = s;
        nodes_[s.child].slot = idx;
        ++table_live_;
    }
    full_dirty_ = true;
    dirty_slots_.clear();
}
void TokenTreeIndex::table_insert(uint32_t parent, const uint32_t* page, uint32_t child) {
    if ((table_live_ + table_tombs_ + 1) * 2 > table_.size()) {
        uint32_t cap = (uint32_t)table_.size();
        while ((table_live_ + 1) * 4 > cap) cap *= 2;
        table_rebuild(cap);
    }
    const uint64_t h = key_of(parent, page);
    uint32_t idx = (uint32_t)(h >> 32) & mask_;
    int64_t tomb = -1;
    while (table_[idx].key != 0) {
        if (table_[idx].child == kTombChild && tomb < 0) tomb = idx;
        idx = (idx + 1) & mask_;
    }
    if (tomb >= 0) { idx = (uint32_t)tomb; --table_tombs_; }
    table_[idx] = ChildSlot{h, parent, child};
    nodes_[child].slot = idx;
    ++table_live_;
    mark_slot(idx);
}
void TokenTreeIndex::table_erase(uint32_t parent, const uint32_t* page) {
    int64_t s = find_child(parent, page);
    if (s < 0) return;
    if (nodes_[table_[(size_t)s].child].slot == (uint32_t)s) nodes_[table_[(size_t)s].child].slot = kNoNode;
    table_[(size_t)s].child = kTombChild;
    --table_live_;
    ++table_tombs_;
    mark_slot((uint32_t)s);
}

uint32_t TokenTreeIndex::new_node(uint64_t off, uint32_t len, uint32_t parent, bool draw_ts) {
    uint32_t id;
    if (!free_nodes_.empty()) { id = free_nodes_.back(); free_nodes_.pop_back(); nodes_[id] = Node(); }
    else {
        id = (uint32_t)nodes_.size();
        size_t before = nodes_.capacity();
        nodes_.emplace_back();
        if (nodes_.capacity() != before) full_dirty_ = true;   // device header array must grow too
    }
    Node& nd = nodes_[id];
    nd.label_off = off; nd.label_len = len; nd.parent = parent;
    nd.creation_time = draw_ts ? next_ts() : 0;   // Node::new draws a timestamp (token_tree.rs:219)
    ++live_nodes_;
    mark_node(id);
    return id;
}
void TokenTreeIndex::free_node(uint32_t id) {
    nodes_[id].alive = false;
    nodes_[id].tenants.clear();
    nodes_[id].kids.clear();
    free_nodes_.push_back(id);
    --live_nodes_;
    mark_node(id);
}
bool TokenTreeIndex::has_tenant(const Node& nd, uint32_t t) const {
    for (auto& kv : nd.tenants) if (kv.first == t) return true;
    return false;
}
void TokenTreeIndex::set_tenant_ts(Node& nd, uint32_t t, uint64_t ts) {
    for (auto& kv : nd.tenants) if (kv.first == t) { kv.second = ts; return; }
    nd.tenants.emplace_back(t, ts);
}
// Node::touch_tenant (token_tree.rs:291-314)
void TokenTreeIndex::touch(uint32_t node, uint32_t tenant) {
    const uint64_t ts = next_ts();
    Node& nd = nodes_[node];
    if (policy_ == EVP_LFU) ++nd.hit_count;
    set_tenant_ts(nd, tenant, ts);
    if ((ts & 0xF) == 0) nd.last_tenant = (int32_t)tenant;
    mark_node(node);
}
// Node::get_any_tenant (token_tree.rs:268-284); the DashMap-order fallback is the lexicographically smallest tenant
int32_t TokenTreeIndex::any_tenant(uint32_t node) const {
    const Node& nd = nodes_[node];
    if (nd.last_tenant >= 0 && has_tenant(nd, (uint32_t)nd.last_tenant)) return nd.last_tenant;
    int32_t best = -1;
    for (auto& kv : nd.tenants) if (best < 0 || tenants_->rank[kv.first] < tenants_->rank[(uint32_t)best]) best = (int32_t)kv.first;
    return best;
}
void TokenTreeIndex::refresh_all_any_tenant() { full_dirty_ = true; }

size_t TokenTreeIndex::tenant_token_size(uint32_t tenant) const {
    return tenant < tenant_tokens_.size() ? tenant_tokens_[tenant] : 0;
}

// TokenTree::insert_tokens (token_tree.rs:401-609)
void TokenTreeIndex::insert_tokens(const uint32_t* toks, size_t n, uint32_t tenant) {
    const size_t aligned = (n / kPage) * kPage;
    if (aligned == 0) return;
    if (tenant >= tenant_known_.size()) { tenant_known_.resize(tenant + 1, 0); tenant_tokens_.resize(tenant + 1, 0); root_has_.resize(tenant + 1, 0); }
    tenant_known_[tenant] = 1;   // token counter (:418-420)
    if (!root_has_[tenant]) {    // root entry (:412-416), on every insert: eviction may have removed it since the first one
        root_has_[tenant] = 1;
        nodes_[0].tenants.emplace_back(tenant, 0);
    }
    const uint32_t* rem = toks;
    size_t rem_len = aligned;
    uint32_t cur = 0;
    size_t added = 0;
    auto append = [&](const uint32_t* t, size_t len) -> uint64_t {
        uint64_t off = tokens_.size();
        tokens_.insert(tokens_.end(), t, t + len);
        return off;
    };
    while (rem_len >= kPage) {
        const int64_t slot = find_child(cur, rem);
        if (slot < 0) {   // vacant: one leaf holding ALL remaining tokens (:441-448)
            const uint64_t off = append(rem, rem_len);
            const uint32_t nn = new_node(off, (uint32_t)rem_len, cur, true);
            touch(nn, tenant);
            table_insert(cur, rem, nn);
            nodes_[cur].kids.push_back(nn);
            added += rem_len;
            break;
        }
        const uint32_t child = table_[(size_t)slot].child;
        const uint32_t child_len = nodes_[child].label_len;
        size_t common = 0;
        {   // only whole equal pages count (:455-463), so compare page by page
            const uint32_t* lab = label(nodes_[child]);
            const size_t lim = std::min<size_t>(rem_len, child_len) / kPage * kPage;
            while (common < lim && memcmp(rem + common, lab + common, kPage * 4) == 0) common += kPage;
        }
        if (common == 0) break;
        if (common == child_len) {   // full edge match → descend; `advance` is counted even for an existing owner (:467-474)
            touch(child, tenant);
            added += common;
            rem += common; rem_len -= common;
            cur = child;
            continue;
        }
        // split at a page boundary: NEW intermediate holds the prefix and clones the child's metadata (:497-507, :545-555)
        const bool owned = has_tenant(nodes_[child], tenant);
        const uint64_t child_off = nodes_[child].label_off;
        const uint32_t mid = new_node(child_off, (uint32_t)common, cur, false);
        nodes_[mid].tenants = nodes_[child].tenants;
        nodes_[mid].last_tenant = nodes_[child].last_tenant;
        nodes_[mid].hit_count = nodes_[child].hit_count;
        nodes_[mid].creation_time = nodes_[child].creation_time;
        nodes_[mid].priority = nodes_[child].priority;
        nodes_[mid].split_epoch = nodes_[child].split_epoch = chunk_epoch_;
        nodes_[child].label_off = child_off + common;
        nodes_[child].label_len = child_len - (uint32_t)common;
        nodes_[child].parent = mid;
        mark_node(child);
        nodes_[mid].kids.push_back(child);
        for (auto& k : nodes_[cur].kids) if (k == child) { k = mid; break; }
        table_[(size_t)slot].child = mid;                          // same page key, now → intermediate
        nodes_[mid].slot = (uint32_t)slot;
        mark_slot((uint32_t)slot);
        table_insert(mid, tokens_.data() + child_off + common, child);
        if (common >= rem_len) {                                   // input is a prefix of the edge (:475-523)
            touch(mid, tenant);
            added += owned ? 0 : common;
        } else {                                                   // diverge: new branch for the rest of the input (:524-585)
            const uint32_t* nr = rem + common;
            const size_t nr_len = rem_len - common;
            size_t branch = 0;
            if (nr_len >= kPage) {
                const uint64_t off = append(nr, nr_len);
                const uint32_t nb = new_node(off, (uint32_t)nr_len, mid, true);
                touch(nb, tenant);
                table_insert(mid, nr, nb);
                nodes_[mid].kids.push_back(nb);
                branch = nr_len;
            }
            touch(mid, tenant);
            added += branch + (owned ? 0 : common);
        }
        break;
    }
    if (added > 0) tenant_tokens_[tenant] += added;
}

// TokenTree::match_prefix_with_counts (token_tree.rs:615-740), host walk
TreeMatch TokenTreeIndex::match_prefix_host(const uint32_t* toks, size_t n, bool do_touch) {
    TreeMatch r{-1, 0, (uint32_t)n, {}, {}};
    const size_t aligned = (n / kPage) * kPage;
    if (aligned == 0) { r.tenant = any_tenant(0); return r; }
    const uint32_t* rem = toks;
    size_t rem_len = aligned;
    uint32_t cur = 0;
    while (rem_len >= kPage) {
        const int64_t slot = find_child(cur, rem);
        if (slot < 0) break;
        const uint32_t child = table_[(size_t)slot].child;
        const uint32_t* lab = label(nodes_[child]);
        const size_t lim = std::min<size_t>(rem_len, nodes_[child].label_len);
        size_t m = 0;
        while (m < lim && rem[m] == lab[m]) ++m;
        m = (m / kPage) * kPage;
        if (m == 0) break;
        const int32_t t = any_tenant(child);
        if (t < 0) break;
        if (do_touch) touch(child, (uint32_t)t);
        r.matched += (uint32_t)m;
        r.tenant = t;
        r.path.push_back(child);
        r.path_tenants.push_back(t);
        if (m < nodes_[child].label_len) break;
        rem += m; rem_len -= m;
        cur = child;
    }
    return r;
}
void TokenTreeIndex::apply_match_touches(const uint32_t* path, const int32_t* path_tenants, uint32_t path_len) {
    for (uint32_t d = 0; d < path_len; ++d) if (path_tenants[d] >= 0) touch(path[d], (uint32_t)path_tenants[d]);
}
void TokenTreeIndex::apply_match_touches(const uint32_t* path, uint32_t path_len) {
    for (uint32_t d = 0; d < path_len; ++d) {
        const int32_t t = any_tenant(path[d]);
        if (t >= 0) touch(path[d], (uint32_t)t);
    }
}

// ---- eviction (token_tree.rs:763-1024) ----
void TokenTreeIndex::evict_tenant(uint32_t tenant, size_t max_tokens) {
    const size_t current = tenant_token_size(tenant);
    if (current <= max_tokens) return;
    const size_t to_evict = current - max_tokens;
    size_t evicted = 0;
    auto first_page_less = [&](uint32_t a, uint32_t b) {
        return std::lexicographical_compare(label(nodes_[a]), label(nodes_[a]) + kPage, label(nodes_[b]), label(nodes_[b]) + kPage);
    };
    auto tenant_ts = [&](uint32_t node, uint64_t& ts) -> bool {
        for (auto& kv : nodes_[node].tenants) if (kv.first == tenant) { ts = kv.second; return true; }
        return false;
    };
    auto is_leaf_for = [&](uint32_t node) {
        uint64_t ts;
        if (!tenant_ts(node, ts)) return false;
        for (uint32_t k : nodes_[node].kids) if (has_tenant(nodes_[k], tenant)) return false;
        return true;
    };
    auto prio = [&](uint32_t node, uint64_t ts) -> std::pair<int64_t, uint64_t> {
        const Node& nd = nodes_[node];
        switch (policy_) {
            case EVP_LRU: return {(int64_t)ts, 0};
            case EVP_LFU: return {(int64_t)nd.hit_count, ts};
            case EVP_FIFO: return {(int64_t)nd.creation_time, 0};
            case EVP_MRU: return {(int64_t)(0 - ts), 0};
            case EVP_FILO: return {(int64_t)(0 - nd.creation_time), 0};
            case EVP_PRIORITY: return {(int64_t)nd.priority, ts};
        }
        return {0, 0};
    };
    // collect_tenant_leaves: post-order DFS, children in lexicographic page-key order (:866-895)
    std::vector<std::pair<uint32_t, uint64_t>> leaves;
    {
        struct Frame { uint32_t node; std::vector<uint32_t> kids; size_t next; bool child_has; };
        std::vector<Frame> st;
        auto push = [&](uint32_t node) {
            Frame f{node, nodes_[node].kids, 0, false};
            std::sort(f.kids.begin(), f.kids.end(), first_page_less);
            for (uint32_t k : f.kids) if (has_tenant(nodes_[k], tenant)) f.child_has = true;
            st.push_back(std::move(f));
        };
        push(0);
        while (!st.empty()) {
            Frame& f = st.back();
            if (f.next < f.kids.size()) { uint32_t k = f.kids[f.next++]; push(k); continue; }
            uint64_t ts;
            if (f.node != 0 && !f.child_has && tenant_ts(f.node, ts)) leaves.push_back({f.node, ts});
            st.pop_back();
        }
    }
    typedef std::pair<std::pair<int64_t, uint64_t>, size_t> Item;
    std::priority_queue<Item, std::vector<Item>, std::greater<Item>> heap;
    std::vector<uint32_t> leaf_nodes;
    for (auto& l : leaves) { heap.push({prio(l.first, l.second), leaf_nodes.size()}); leaf_nodes.push_back(l.first); }
    std::vector<uint32_t> graveyard;
    while (evicted < to_evict && !heap.empty()) {
        const uint32_t node = leaf_nodes[heap.top().second];
        heap.pop();
        // remove_tenant_and_cleanup (:922-985)
        Node& nd = nodes_[node];
        bool had = false;
        for (size_t i = 0; i < nd.tenants.size(); ++i) if (nd.tenants[i].first == tenant) { nd.tenants.erase(nd.tenants.begin() + i); had = true; break; }
        if (!had) continue;
        if (node == 0) root_has_[tenant] = 0;
        mark_node(node);
        evicted += nd.label_len;
        uint32_t cur = node;
        int64_t promoted = -1;
        uint64_t promoted_ts = 0;
        for (;;) {
            Node& c = nodes_[cur];
            const bool empty = c.tenants.empty() && c.kids.empty();
            if (!empty) {
                if (promoted < 0 && is_leaf_for(cur)) { promoted = cur; tenant_ts(cur, promoted_ts); }
                break;
            }
            const uint32_t parent = c.parent;
            if (parent == kNoNode || cur == 0) break;
            table_erase(parent, label(c));
            auto& pk = nodes_[parent].kids;
            pk.erase(std::remove(pk.begin(), pk.end(), cur), pk.end());
            graveyard.push_back(cur);
            if (promoted < 0 && is_leaf_for(parent)) { promoted = parent; tenant_ts(parent, promoted_ts); }
            cur = parent;
        }
        if (promoted >= 0) { heap.push({prio((uint32_t)promoted, promoted_ts), leaf_nodes.size()}); leaf_nodes.push_back((uint32_t)promoted); }
    }
    for (uint32_t g : graveyard) free_node(g);
    if (tenant < tenant_tokens_.size()) tenant_tokens_[tenant] = tenant_tokens_[tenant] >= evicted ? tenant_tokens_[tenant] - evicted : 0;
}
void TokenTreeIndex::evict_tenant_by_size(size_t max_size) {
    std::vector<uint32_t> over;
    for (uint32_t t = 0; t < tenant_tokens_.size(); ++t) if (tenant_known_[t] && tenant_tokens_[t] > max_size) over.push_back(t);
    std::sort(over.begin(), over.end(), [&](uint32_t a, uint32_t b) { return tenants_->names[a] < tenants_->names[b]; });
    for (uint32_t t : over) evict_tenant(t, max_size);
}
void TokenTreeIndex::clear() {
    nodes_.resize(1);
    nodes_[0].tenants.clear();
    nodes_[0].kids.clear();
    free_nodes_.clear();
    live_nodes_ = 0;
    tokens_.clear();
    uploaded_tokens_ = 0;
    table_.assign(1024, ChildSlot{0, 0, 0});
    mask_ = 1023;
    table_live_ = table_tombs_ = 0;
    tenant_tokens_.clear(); tenant_known_.clear(); root_has_.clear();
    full_dirty_ = true;
    dirty_nodes_.clear(); dirty_slots_.clear();
}
void TokenTreeIndex::entries(std::vector<std::pair<std::vector<uint32_t>, std::vector<std::pair<uint32_t, uint64_t>>>>& out) const {
    auto first_page_less = [&](uint32_t a, uint32_t b) {
        return std::lexicographical_compare(label(nodes_[a]), label(nodes_[a]) + kPage, label(nodes_[b]), label(nodes_[b]) + kPage);
    };
    std::vector<uint32_t> path;
    struct Rec { const TokenTreeIndex* self; decltype(first_page_less)& less; std::vector<uint32_t>& path; decltype(out)& out;
        void walk(uint32_t node) {
            const Node& nd = self->nodes_[node];
            if (!nd.tenants.empty()) {
                auto ts = nd.tenants;
                std::sort(ts.begin(), ts.end(), [&](auto& a, auto& b) { return self->tenants_->names[a.first] < self->tenants_->names[b.first]; });
                out.push_back({path, ts});
            }
            std::vector<uint32_t> kids = nd.kids;
            std::sort(kids.begin(), kids.end(), less);
            for (uint32_t k : kids) {
                size_t before = path.size();
                const Node& c = self->nodes_[k];
                path.insert(path.end(), self->label(c), self->label(c) + c.label_len);
                walk(k);
                path.resize(before);
            }
        } } rec{this, first_page_less, path, out};
    rec.walk(0);
}

// =================================================================================================================
// device mirror
// =================================================================================================================
namespace {
__global__ void scatter32_kernel(uint4* __restrict__ dst, const uint32_t* __restrict__ idx, const uint4* __restrict__ src, uint32_t n) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) { const size_t d = (size_t)idx[t] * 2; dst[d] = src[(size_t)t * 2]; dst[d + 1] = src[(size_t)t * 2 + 1]; }
}
}  // namespace

TreeSlot TokenTreeIndex::device_slot(uint32_t i) const {
    const ChildSlot& c = table_[i];
    TreeSlot t{c.key, c.parent, c.child, 0, 0, -1};
    if (c.key != 0 && c.child < kTombChild) {
        const Node& nd = nodes_[c.child];
        t.label_off = nd.label_off;
        t.label_len = nd.alive ? nd.label_len : 0;
        t.any_tenant = nd.alive ? any_tenant(c.child) : -1;
    }
    return t;
}

TokenTreeView TokenTreeIndex::flush(cudaStream_t stream, uint64_t* launches) {
    if (!device_enabled) throw Error(SMGX_DEVICE_ERROR, "policy was created with device_id = -1 (host mirror only): no GPU path, no CPU fallback");
    if (tenants_version_seen != tenants_->version) { full_dirty_ = true; tenants_version_seen = tenants_->version; }
    // token arena: append-only
    if (tokens_.size() * 4 > d_tokens_.cap) {
        if (stage_pending_) { SMGX_CUDA(cudaEventSynchronize(stage_done_)); stage_pending_ = false; }
        SMGX_CUDA(cudaDeviceSynchronize());
        d_tokens_.reserve(std::max<size_t>(tokens_.capacity(), 1024) * 4);
        uploaded_tokens_ = 0;
    }
    if (uploaded_tokens_ < tokens_.size()) {
        SMGX_CUDA(cudaMemcpyAsync(d_tokens_.as<uint32_t>() + uploaded_tokens_, tokens_.data() + uploaded_tokens_,
                                  (tokens_.size() - uploaded_tokens_) * 4, cudaMemcpyHostToDevice, stream));
        uploaded_tokens_ = tokens_.size();
    }
    // a node whose header changed dirties the slot that points at it
    for (uint32_t id : dirty_nodes_) if (id < nodes_.size() && nodes_[id].slot != kNoNode) mark_slot(nodes_[id].slot);
    dirty_nodes_.clear();
    if (!full_dirty_ && dirty_slots_.size() > table_.size() / 8) full_dirty_ = true;
    if (full_dirty_) {
        if (stage_pending_) { SMGX_CUDA(cudaEventSynchronize(stage_done_)); stage_pending_ = false; }
        SMGX_CUDA(cudaDeviceSynchronize());
        std::vector<TreeSlot> dev(table_.size());
        for (uint32_t i = 0; i < table_.size(); ++i) dev[i] = device_slot(i);
        d_table_.reserve(table_.size() * sizeof(TreeSlot));
        SMGX_CUDA(cudaMemcpyAsync(d_table_.ptr, dev.data(), dev.size() * sizeof(TreeSlot), cudaMemcpyHostToDevice, stream));
        SMGX_CUDA(cudaStreamSynchronize(stream));   // `dev` is a temporary
        full_dirty_ = false;
        dirty_slots_.clear();
    } else if (!dirty_slots_.empty()) {
        if (!stage_done_) SMGX_CUDA(cudaEventCreateWithFlags(&stage_done_, cudaEventDisableTiming));
        if (stage_pending_) { SMGX_CUDA(cudaEventSynchronize(stage_done_)); stage_pending_ = false; }
        const size_t ns = dirty_slots_.size();   // unique by construction (mark_slot stamps)
        const size_t off_r = ((ns * 4 + 15) / 16) * 16, total = off_r + ns * 32;
        stage_.reserve(total);
        d_stage_.reserve(total);
        char* st = stage_.as<char>();
        memcpy(st, dirty_slots_.data(), ns * 4);
        for (size_t i = 0; i < ns; ++i) { const TreeSlot t = device_slot(dirty_slots_[i]); memcpy(st + off_r + i * 32, &t, 32); }
        SMGX_CUDA(cudaMemcpyAsync(d_stage_.ptr, st, total, cudaMemcpyHostToDevice, stream));
        char* ds = d_stage_.as<char>();
        scatter32_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, stream>>>(d_table_.as<uint4>(), (const uint32_t*)ds, (const uint4*)(ds + off_r), (uint32_t)ns);
        ++*launches;
        SMGX_CUDA(cudaGetLastError());
        SMGX_CUDA(cudaEventRecord(stage_done_, stream));
        stage_pending_ = true;
        dirty_slots_.clear();
    }
    if (++flush_gen_ == 0) { flush_gen_ = 1; std::fill(slot_stamp_.begin(), slot_stamp_.end(), 0u); }
    return TokenTreeView{d_tokens_.as<uint32_t>(), d_table_.as<TreeSlot>(), mask_};
}

// =================================================================================================================
// K2a + K3: longest page-aligned prefix match + pick, one warp per request
// =================================================================================================================
namespace {
constexpr unsigned FULLM = 0xffffffffu;

constexpr uint32_t kWin = 512;   // request tokens staged per warp in shared memory (one BASELINE config-2 request)

// One warp per request.  At the H100's HBM roofline an SM sub-partition has ≈1260 issue slots per 512-token request (4032 B at 3.35 TB/s,
// 528 sub-partitions at 1.98 GHz), so the walk is
// written for few instructions as much as for few dependent reads:
//   * the request is staged in shared memory with every load issued at once (off the hash → probe → label chain);
//   * the page key is two 32-bit multilinear sums, one redux.sync each;
//   * the child's header rides in the 32 B slot: a probe hit needs no second dependent read;
//   * labels are compared 256 tokens per round as OR-of-XORs; the exact mismatch position is only computed when there is one.
template <int TILE, class Tile>
__device__ __forceinline__ void tree_walk_request(const Tile& tile, uint32_t* __restrict__ win, const TokenTreeView& tv, const FleetView& f,
                                                  const int32_t* __restrict__ slice_of_tenant, const uint8_t* __restrict__ flags, uint32_t n_tenants,
                                                  const TreeSelectArgs& a, uint32_t r) {
    static_assert(TILE == 32, "the walk uses one warp per request");
    const int rank = (int)tile.thread_rank();
    const uint32_t off = a.offsets[r], ntok = a.offsets[r + 1] - off;
    const uint32_t* tok = a.tokens + off;
    const uint32_t aligned = (ntok / kPage) * kPage;
    const uint32_t mult = rank < 16 ? page_mult1((uint32_t)rank) : page_mult2((uint32_t)rank - 16);
    const uint32_t salt_add = rank < 16 ? 1u : 0u, salt_xor = rank < 16 ? 0u : 0x9E3779B9u;
    const bool vec_ok = (reinterpret_cast<uintptr_t>(tok) & 15) == 0;
    uint32_t wbase = 0, wend = 0;
    auto load_window = [&](uint32_t start) {   // stage request tokens [start, start + kWin)
        __syncwarp();
        wbase = start;
        wend = min(start + kWin, aligned);
        const uint32_t n = wend - wbase;
        if (vec_ok) for (uint32_t j = (uint32_t)rank * 4; j < n; j += 128) *reinterpret_cast<uint4*>(win + j) = *reinterpret_cast<const uint4*>(tok + wbase + j);
        else for (uint32_t j = rank; j < n; j += 32) win[j] = tok[wbase + j];
        __syncwarp();
    };
    load_window(0);

    uint32_t cur = 0, pos = 0, matched = 0, depth = 0;
    int32_t tenant = -1;
    while (aligned - pos >= kPage) {
        if (pos < wbase || pos + kPage > wend) load_window(pos);
        // key of (cur, next 16 tokens): lanes 0-15 feed the first sum, lanes 16-31 the second
        const uint32_t t = win[pos - wbase + (rank & 15)];
        const uint32_t term = ((t + salt_add) ^ salt_xor) * mult;
        const uint32_t h1 = __reduce_add_sync(FULLM, rank < 16 ? term : 0u);
        const uint32_t h2 = __reduce_add_sync(FULLM, rank < 16 ? 0u : term);
        const uint64_t key = page_finish(h1, h2, cur);
        uint32_t idx = (uint32_t)(key >> 32) & tv.child_mask;
        uint32_t child = kNoNode, m = 0, label_len = 0;
        int32_t any = -1;
        for (;;) {   // warp-uniform probe
            const uint4* sp = reinterpret_cast<const uint4*>(tv.slots + idx);
            const uint4 sa = __ldg(sp);
            const uint64_t skey = ((uint64_t)sa.y << 32) | sa.x;
            if (skey == 0) break;
            if (skey == key && sa.z == cur && sa.w < kTombChild) {
                const uint4 sb = __ldg(sp + 1);   // same 32 B sector as sa
                const uint64_t label_off = ((uint64_t)sb.y << 32) | sb.x;
                label_len = sb.z; any = (int32_t)sb.w;
                const uint32_t L = min(label_len, aligned - pos);
                const uint32_t* lab = tv.tokens + label_off;   // always 16 B aligned: the arena only grows and splits by whole pages
                uint32_t common = L;
                for (uint32_t c = 0; c < L; c += 256) {
                    if (pos + c < wbase || pos + c + min(256u, L - c) > wend) load_window(pos + c);
                    const uint32_t j0 = c + (uint32_t)rank * 4, j1 = j0 + 128;
                    uint32_t d0 = 0, d1 = 0;
                    if (j0 < L) {
                        const uint4 x = __ldg(reinterpret_cast<const uint4*>(lab + j0)), y = *reinterpret_cast<const uint4*>(win + (pos + j0 - wbase));
                        d0 = (x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w);
                    }
                    if (j1 < L) {
                        const uint4 x = __ldg(reinterpret_cast<const uint4*>(lab + j1)), y = *reinterpret_cast<const uint4*>(win + (pos + j1 - wbase));
                        d1 = (x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w);
                    }
                    const unsigned m0 = __ballot_sync(FULLM, d0 != 0), m1 = __ballot_sync(FULLM, d1 != 0);
                    if (m0 | m1) {   // first differing token: only now look inside the quad (re-read, it is in cache)
                        const bool lo = m0 != 0;
                        const int src = __ffs((int)(lo ? m0 : m1)) - 1;
                        const uint32_t jq = c + (lo ? 0u : 128u) + (uint32_t)src * 4;
                        const uint4 x = __ldg(reinterpret_cast<const uint4*>(lab + jq)), y = *reinterpret_cast<const uint4*>(win + (pos + jq - wbase));
                        common = jq + (x.x != y.x ? 0u : x.y != y.y ? 1u : x.z != y.z ? 2u : 3u);
                        break;
                    }
                }
                m = (common / kPage) * kPage;
                if (m > 0) { child = sa.w; break; }   // m == 0: different page under the same 64-bit key — keep probing
                if (pos < wbase || pos + kPage > wend) load_window(pos);
            }
            idx = (idx + 1) & tv.child_mask;
        }
        if (child == kNoNode) break;
        if (any < 0) break;                            // node without tenants ends the walk before being counted (:682-683)
        matched += m;
        tenant = any;
        if (rank == 0 && depth < kPathCap && a.out_path) {
            a.out_path[(size_t)r * kPathCap + depth] = child;
            a.out_path_tenant[(size_t)r * kPathCap + depth] = any;
        }
        ++depth;
        if (m < label_len) break;                      // partial edge match (:691-696)
        pos += m;
        cur = child;
    }
    if (rank != 0) return;
    if (a.out_path_len) a.out_path_len[r] = depth;
    if (a.out_tenant) a.out_tenant[r] = tenant;
    int32_t out = -1;
    uint32_t branch = SMGX_BR_NO_HEALTHY;
    if (a.decide) {
        const FleetDerived fd = *f.derived;
        if (fd.n_healthy == 0) {
        } else if (fd.imbalanced) {
            out = fd.min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD;
        } else {
            // match_rate = matched as f32 / input as f32 (UNALIGNED input length), strict > (cache_aware.rs:848-854)
            const float rate = ntok == 0 ? 0.0f : __fdiv_rn(__uint2float_rn(matched), __uint2float_rn(ntok));
            if (rate > a.cache_threshold) {
                int32_t sl = (tenant >= 0 && (uint32_t)tenant < n_tenants) ? slice_of_tenant[tenant] : -1;
                if (sl >= 0 && (flags[sl] & 1)) { out = sl; branch = SMGX_BR_TREE_MATCH; }         // .filter(is_healthy) only (:859)
                else { out = fd.first_healthy; branch = SMGX_BR_TREE_FALLBACK_FIRST_HEALTHY; }   // (:892-894)
            } else { out = fd.min_load_idx; branch = SMGX_BR_TREE_MIN_LOAD; }
        }
    }
    a.out_idx[r] = out;
    if (a.out_info) {
        smgx_decision_info di;
        di.matched = matched; di.input = ntok; di.branch = (uint8_t)branch;
        di.nodes = (uint8_t)min(depth, 255u);
        di.reserved[0] = di.reserved[1] = 0;
        a.out_info[r] = di;
    }
}

// one tile per request of one segment (the select path: first/count of one batch)
template <int TILE>
__global__ void __launch_bounds__(256, 5) tree_select_kernel(TokenTreeView tv, FleetView f, const int32_t* __restrict__ slice_of_tenant,
                                                          const uint8_t* __restrict__ flags, uint32_t n_tenants, TreeSelectArgs a) {
    namespace cg = cooperative_groups;
    const auto tile = cg::tiled_partition<TILE>(cg::this_thread_block());
    __shared__ __align__(16) uint32_t win_all[8][kWin];
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) / TILE;
    if (w >= a.count) return;
    tree_walk_request<TILE>(tile, win_all[threadIdx.x >> 5], tv, f, slice_of_tenant, flags, n_tenants, a, a.first + w);
}

}  // namespace

void launch_tree_select(const TokenTreeView& tv, const FleetView& fleet, const int32_t* d_slice_of_tenant, const uint8_t* d_flags,
                        uint32_t n_tenants, const TreeSelectArgs& a, cudaStream_t stream) {
    if (a.count == 0) return;
    tree_select_kernel<32><<<(unsigned)(((uint64_t)a.count * 32 + 255) / 256), 256, 0, stream>>>(tv, fleet, d_slice_of_tenant, d_flags, n_tenants, a);
    SMGX_CUDA(cudaGetLastError());
}

}  // namespace smgx
