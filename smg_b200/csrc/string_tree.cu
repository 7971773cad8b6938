// K2c — char-level string tree: host tree + device mirror + the match/decide kernel.  See string_tree.h.
#include "string_tree.h"

#include <memory>

#include <algorithm>
#include <cstring>
#include <queue>

#include "kernels.h"

namespace smgx {

// =================================================================================================================
// host tree
// =================================================================================================================
StringTreeIndex::StringTreeIndex(TenantTable* tenants, uint64_t* epoch) : tenants_(tenants), epoch_(epoch) {
    nodes_.emplace_back();
    table_.assign(1024, StrChildSlot{0, 0, 0});
    mask_ = 1023;
}
StringTreeIndex::~StringTreeIndex() {
    d_bytes_.release(); d_table_.release(); d_stage_.release(); stage_.release();
    if (stage_done_) cudaEventDestroy(stage_done_);
}

bool StringTreeIndex::valid_utf8(const uint8_t* s, size_t n) {   // Rust `&str` is valid UTF-8 by construction; the C ABI checks
    size_t i = 0;
    while (i < n) {
        const uint8_t c = s[i];
        size_t len;
        if (c < 0x80) { ++i; continue; }
        else if (c >= 0xC2 && c <= 0xDF) len = 2;
        else if (c >= 0xE0 && c <= 0xEF) len = 3;
        else if (c >= 0xF0 && c <= 0xF4) len = 4;
        else return false;
        if (i + len > n) return false;
        for (size_t k = 1; k < len; ++k) if ((s[i + k] & 0xC0) != 0x80) return false;
        if (len == 3) {
            if (c == 0xE0 && s[i + 1] < 0xA0) return false;
            if (c == 0xED && s[i + 1] > 0x9F) return false;   // surrogates
        } else if (len == 4) {
            if (c == 0xF0 && s[i + 1] < 0x90) return false;
            if (c == 0xF4 && s[i + 1] > 0x8F) return false;
        }
        i += len;
    }
    return true;
}

int64_t StringTreeIndex::find_child(uint32_t parent, uint32_t cp) const {
    const uint64_t key = str_child_key(parent, cp);
    uint32_t idx = str_child_home(key) & mask_;
    for (;;) {
        const StrChildSlot& s = table_[idx];
        if (s.key == 0) return -1;
        if (s.key == key && s.child < kTombChild) return idx;
        idx = (idx + 1) & mask_;
    }
}
void StringTreeIndex::table_rebuild(uint32_t cap) {
    std::vector<StrChildSlot> old;
    old.swap(table_);
    table_.assign(cap, StrChildSlot{0, 0, 0});
    mask_ = cap - 1;
    table_live_ = table_tombs_ = 0;
    for (const StrChildSlot& s : old) {
        if (s.key == 0 || s.child >= kTombChild) continue;
        uint32_t idx = str_child_home(s.key) & mask_;
        while (table_[idx].key != 0) idx = (idx + 1) & mask_;
        table_[idx] = s;
        nodes_[s.child].slot = idx;
        ++table_live_;
    }
    full_dirty_ = true;
    dirty_slots_.clear();
}
void StringTreeIndex::table_insert(uint32_t parent, uint32_t cp, uint32_t child) {
    if ((table_live_ + table_tombs_ + 1) * 2 > table_.size()) {
        uint32_t cap = (uint32_t)table_.size();
        while ((table_live_ + 1) * 4 > cap) cap *= 2;
        table_rebuild(cap);
    }
    const uint64_t key = str_child_key(parent, cp);
    uint32_t idx = str_child_home(key) & mask_;
    int64_t tomb = -1;
    while (table_[idx].key != 0) {
        if (table_[idx].child == kTombChild && tomb < 0) tomb = idx;
        idx = (idx + 1) & mask_;
    }
    if (tomb >= 0) { idx = (uint32_t)tomb; --table_tombs_; }
    table_[idx] = StrChildSlot{key, child, 0};
    nodes_[child].slot = idx;
    ++table_live_;
    mark_slot(idx);
}
void StringTreeIndex::table_set(uint32_t parent, uint32_t cp, uint32_t child) {
    const int64_t s = find_child(parent, cp);
    if (s < 0) { table_insert(parent, cp, child); return; }
    table_[(size_t)s].child = child;
    nodes_[child].slot = (uint32_t)s;
    mark_slot((uint32_t)s);
}
void StringTreeIndex::table_erase(uint32_t parent, uint32_t cp) {
    const int64_t s = find_child(parent, cp);
    if (s < 0) return;
    if (nodes_[table_[(size_t)s].child].slot == (uint32_t)s) nodes_[table_[(size_t)s].child].slot = kNoNode;
    table_[(size_t)s].child = kTombChild;
    --table_live_;
    ++table_tombs_;
    mark_slot((uint32_t)s);
}

uint32_t StringTreeIndex::new_node(uint64_t off, uint32_t bytes, uint32_t chars, uint32_t parent, uint32_t first_cp) {
    uint32_t id;
    if (!free_nodes_.empty()) { id = free_nodes_.back(); free_nodes_.pop_back(); nodes_[id] = Node(); }
    else {
        id = (uint32_t)nodes_.size();
        const size_t before = nodes_.capacity();
        nodes_.emplace_back();
        if (nodes_.capacity() != before) full_dirty_ = true;
    }
    Node& nd = nodes_[id];
    nd.label_off = off; nd.label_bytes = bytes; nd.label_chars = chars; nd.parent = parent; nd.first_cp = first_cp;
    ++live_nodes_;
    mark_node(id);
    return id;
}
void StringTreeIndex::free_node(uint32_t id) {
    Node& nd = nodes_[id];
    nd.alive = false; nd.tenants.clear(); nd.kids.clear(); nd.last_tenant = -1;
    free_nodes_.push_back(id);
    --live_nodes_;
    mark_node(id);
}
int64_t StringTreeIndex::find_tenant(const Node& nd, uint32_t t) {
    for (size_t i = 0; i < nd.tenants.size(); ++i) if (nd.tenants[i].first == t) return (int64_t)i;
    return -1;
}
void StringTreeIndex::set_tenant(Node& nd, uint32_t t, uint64_t ts) {
    const int64_t i = find_tenant(nd, t);
    if (i >= 0) nd.tenants[(size_t)i].second = ts; else nd.tenants.emplace_back(t, ts);
}
void StringTreeIndex::erase_tenant(Node& nd, uint32_t t) {
    const int64_t i = find_tenant(nd, t);
    if (i >= 0) nd.tenants.erase(nd.tenants.begin() + i);
}
// tenant the match reports for a node (:598-627): valid cached last_tenant, else "first in DashMap order" = smallest name
int32_t StringTreeIndex::any_tenant(const Node& nd) const {
    if (cache_valid(nd)) return nd.last_tenant;
    int32_t best = -1;
    for (auto& kv : nd.tenants) if (best < 0 || tenants_->rank[kv.first] < tenants_->rank[(uint32_t)best]) best = (int32_t)kv.first;
    return best;
}
void StringTreeIndex::kids_insert(Node& nd, uint32_t cp, uint32_t child) {
    auto it = std::lower_bound(nd.kids.begin(), nd.kids.end(), std::make_pair(cp, 0u));
    if (it != nd.kids.end() && it->first == cp) it->second = child; else nd.kids.insert(it, {cp, child});
}
void StringTreeIndex::kids_erase(Node& nd, uint32_t cp) {
    auto it = std::lower_bound(nd.kids.begin(), nd.kids.end(), std::make_pair(cp, 0u));
    if (it != nd.kids.end() && it->first == cp) nd.kids.erase(it);
}

static inline uint32_t count_chars(const uint8_t* s, size_t n) {   // bytes − continuation bytes (10xxxxxx), 8 at a time
    size_t i = 0, cont = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w;
        memcpy(&w, s + i, 8);
        cont += (size_t)__builtin_popcountll((w >> 7) & ~(w >> 6) & 0x0101010101010101ULL);
    }
    for (; i < n; ++i) cont += (s[i] & 0xC0) == 0x80;
    return (uint32_t)(n - cont);
}
// shared prefix of two valid UTF-8 strings, in bytes, ending on a char boundary (shared_prefix_count :311-338)
static inline size_t shared_prefix_bytes(const uint8_t* a, size_t na, const uint8_t* b, size_t nb) {
    const size_t lim = std::min(na, nb);
    size_t i = 0;
    while (i + 8 <= lim) {   // 8 bytes at a time; the first differing byte from the lowest set bit of the XOR (little endian)
        uint64_t x, y;
        memcpy(&x, a + i, 8); memcpy(&y, b + i, 8);
        if (x != y) { i += (size_t)(__builtin_ctzll(x ^ y) >> 3); break; }
        i += 8;
    }
    while (i < lim && a[i] == b[i]) ++i;
    if (i < lim) while (i > 0 && (a[i] & 0xC0) == 0x80) --i;   // mismatch inside a char: back to its first byte
    return i;
}

// Tree::insert_text (string_tree.rs:393-557)
void StringTreeIndex::insert_text(const uint8_t* s, size_t n, uint32_t tenant) {
    if (find_tenant(nodes_[0], tenant) < 0) { nodes_[0].tenants.emplace_back(tenant, 0); mark_node(0); }
    tenant_chars_.emplace(tenant, 0);
    size_t off = 0;
    uint32_t prev = 0;
    while (off < n) {
        uint32_t cl;
        const uint32_t cp = utf8_first(s + off, &cl);
        const int64_t slot = find_child(prev, cp);
        if (slot < 0) {   // vacant: one leaf with the whole remaining text, owned and cached by the inserting tenant (:413-441)
            const uint32_t chars = count_chars(s + off, n - off);
            const uint64_t epoch = next_epoch();
            const uint64_t boff = bytes_.size();
            bytes_.insert(bytes_.end(), s + off, s + n);
            const uint32_t leaf = new_node(boff, (uint32_t)(n - off), chars, prev, cp);
            nodes_[leaf].last_tenant = (int32_t)tenant;
            nodes_[leaf].tenants.emplace_back(tenant, epoch);
            tenant_chars_[tenant] += chars;
            table_insert(prev, cp, leaf);
            kids_insert(nodes_[prev], cp, leaf);
            return;
        }
        const uint32_t m = table_[(size_t)slot].child;
        const size_t shared = shared_prefix_bytes(s + off, n - off, label(nodes_[m]), nodes_[m].label_bytes);
        if (shared < nodes_[m].label_bytes) {   // split: a NEW intermediate takes the shared prefix and clones tenants + cache (:455-510)
            const uint32_t shared_chars = count_chars(s + off, shared);
            const uint64_t moff = nodes_[m].label_off;
            const uint32_t nn = new_node(moff, (uint32_t)shared, shared_chars, prev, cp);
            nodes_[nn].tenants = nodes_[m].tenants;
            nodes_[nn].last_tenant = nodes_[m].last_tenant;
            nodes_[nn].split_epoch = nodes_[m].split_epoch = chunk_epoch_;
            Node& mm = nodes_[m];
            mm.label_off = moff + shared; mm.label_bytes -= (uint32_t)shared; mm.label_chars -= shared_chars; mm.parent = nn;
            uint32_t l2;
            mm.first_cp = utf8_first(label(mm), &l2);
            mark_node(m);
            kids_insert(nodes_[nn], mm.first_cp, m);
            table_set(prev, cp, nn);
            kids_insert(nodes_[prev], cp, nn);
            table_insert(nn, mm.first_cp, m);
            if (find_tenant(nodes_[nn], tenant) < 0) {
                tenant_chars_[tenant] += shared_chars;
                nodes_[nn].tenants.emplace_back(tenant, 0);
            }
            prev = nn;
        } else {
            Node& mm = nodes_[m];
            if (find_tenant(mm, tenant) < 0) {
                tenant_chars_[tenant] += mm.label_chars;
                mm.tenants.emplace_back(tenant, 0);
                mark_node(m);
            }
            prev = m;
        }
        off += shared;
    }
    const uint64_t epoch = next_epoch();
    set_tenant(nodes_[prev], tenant, epoch);
    mark_node(prev);
}

// side effects of Tree::match_prefix_with_counts on the node the walk ended on (:598-637)
void StringTreeIndex::apply_match_effects(uint32_t node, int32_t tenant, bool fill_cache) {
    Node& nd = nodes_[node];
    if (fill_cache) { nd.last_tenant = tenant; mark_node(node); }   // tenant < 0 ("empty") leaves the cache invalid, like caching "empty"
    const uint64_t epoch = next_epoch();
    if ((epoch & 0x7) == 0 && tenant >= 0) set_tenant(nd, (uint32_t)tenant, epoch);
}

// Tree::prefix_match_tenant (:659-720)
std::string StringTreeIndex::prefix_match_tenant(const uint8_t* s, size_t n, int64_t tenant) {
    size_t off = 0;
    uint32_t prev = 0;
    while (off < n) {
        uint32_t cl;
        const uint32_t cp = utf8_first(s + off, &cl);
        const int64_t slot = find_child(prev, cp);
        if (slot < 0) break;
        const uint32_t m = table_[(size_t)slot].child;
        if (tenant < 0 || find_tenant(nodes_[m], (uint32_t)tenant) < 0) break;
        const size_t shared = shared_prefix_bytes(s + off, n - off, label(nodes_[m]), nodes_[m].label_bytes);
        off += shared;
        prev = m;
        if (shared != nodes_[m].label_bytes) break;
    }
    if (tenant >= 0 && find_tenant(nodes_[prev], (uint32_t)tenant) >= 0) set_tenant(nodes_[prev], (uint32_t)tenant, next_epoch());
    return std::string((const char*)s, off);
}

std::vector<uint32_t> StringTreeIndex::leaf_of(uint32_t node) const {
    const Node& nd = nodes_[node];
    std::vector<uint32_t> out;
    for (auto& kv : nd.tenants) {
        bool in_child = false;
        for (auto& k : nd.kids) if (find_tenant(nodes_[k.second], kv.first) >= 0) { in_child = true; break; }
        if (!in_child) out.push_back(kv.first);
    }
    std::sort(out.begin(), out.end(), [&](uint32_t a, uint32_t b) { return tenants_->rank[a] < tenants_->rank[b]; });
    return out;
}

// Tree::evict_tenant_by_size (:745-849): one global min-heap over (epoch) of every tenant-leaf; ties in discovery order
void StringTreeIndex::evict_tenant_by_size(size_t max_size) {
    struct Ent { uint64_t ts, seq; uint32_t tenant, node; };
    auto cmp = [](const Ent& a, const Ent& b) { return a.ts != b.ts ? a.ts > b.ts : a.seq > b.seq; };
    std::priority_queue<Ent, std::vector<Ent>, decltype(cmp)> pq(cmp);
    uint64_t seq = 0;
    auto ts_of = [&](uint32_t node, uint32_t t) { const int64_t i = find_tenant(nodes_[node], t); return i >= 0 ? nodes_[node].tenants[(size_t)i].second : 0; };
    std::vector<uint32_t> stack{0};
    while (!stack.empty()) {
        const uint32_t cur = stack.back(); stack.pop_back();
        for (auto& k : nodes_[cur].kids) stack.push_back(k.second);
        for (uint32_t t : leaf_of(cur)) pq.push(Ent{ts_of(cur, t), seq++, t, cur});
    }
    std::vector<uint32_t> graveyard;
    while (!pq.empty()) {
        const Ent e = pq.top(); pq.pop();
        auto sz = tenant_chars_.find(e.tenant);
        if (sz != tenant_chars_.end() && sz->second <= max_size) continue;
        Node& node = nodes_[e.node];
        bool still_leaf = find_tenant(node, e.tenant) >= 0;
        if (still_leaf) for (auto& k : node.kids) if (find_tenant(nodes_[k.second], e.tenant) >= 0) { still_leaf = false; break; }
        if (!still_leaf) continue;
        const size_t node_len = node.label_chars;
        if (sz != tenant_chars_.end()) sz->second = sz->second >= node_len ? sz->second - node_len : 0;
        erase_tenant(node, e.tenant);
        mark_node(e.node);
        const uint32_t parent = node.parent;
        if (node.kids.empty() && node.tenants.empty() && parent != kNoNode && node.label_bytes > 0) {
            table_erase(parent, node.first_cp);
            kids_erase(nodes_[parent], node.first_cp);
            graveyard.push_back(e.node);
        }
        if (parent != kNoNode && find_tenant(nodes_[parent], e.tenant) >= 0) {
            bool child_has = false;
            for (auto& k : nodes_[parent].kids) if (find_tenant(nodes_[k.second], e.tenant) >= 0) { child_has = true; break; }
            if (!child_has) pq.push(Ent{ts_of(parent, e.tenant), seq++, e.tenant, parent});
        }
    }
    for (uint32_t g : graveyard) free_node(g);
}

size_t StringTreeIndex::tenant_char_size(uint32_t tenant) const {
    auto it = tenant_chars_.find(tenant);
    return it == tenant_chars_.end() ? 0 : it->second;
}
std::map<std::string, size_t> StringTreeIndex::tenant_char_counts() const {
    std::map<std::string, size_t> out;
    for (auto& kv : tenant_chars_) out[tenants_->names[kv.first]] = kv.second;
    return out;
}
std::map<std::string, size_t> StringTreeIndex::used_size_per_tenant() const {
    std::map<std::string, size_t> out;
    for (uint32_t i = 0; i < nodes_.size(); ++i) {
        const Node& nd = nodes_[i];
        if (!nd.alive) continue;
        for (auto& kv : nd.tenants) out[tenants_->names[kv.first]] += nd.label_chars;
    }
    return out;
}
void StringTreeIndex::clear() {
    nodes_.clear(); nodes_.emplace_back();
    free_nodes_.clear(); live_nodes_ = 0;
    bytes_.clear(); uploaded_bytes_ = 0;
    table_.assign(1024, StrChildSlot{0, 0, 0}); mask_ = 1023; table_live_ = table_tombs_ = 0;
    tenant_chars_.clear();
    full_dirty_ = true; dirty_nodes_.clear(); dirty_slots_.clear();
}
void StringTreeIndex::entries(std::vector<std::pair<std::string, std::vector<std::pair<uint32_t, uint64_t>>>>& out) const {
    struct Frame { uint32_t node; size_t path_len; };
    std::string path;
    // explicit pre-order, children in char order
    std::vector<std::pair<uint32_t, size_t>> stack{{0, 0}};
    while (!stack.empty()) {
        auto [id, plen] = stack.back(); stack.pop_back();
        const Node& nd = nodes_[id];
        path.resize(plen);
        path.append((const char*)label(nd), nd.label_bytes);
        if (!nd.tenants.empty()) {
            std::vector<std::pair<uint32_t, uint64_t>> ts(nd.tenants.begin(), nd.tenants.end());
            std::sort(ts.begin(), ts.end(), [&](auto& a, auto& b) { return tenants_->rank[a.first] < tenants_->rank[b.first]; });
            out.push_back({path, ts});
        }
        for (size_t k = nd.kids.size(); k-- > 0;) stack.push_back({nd.kids[k].second, path.size()});
    }
}

// =================================================================================================================
// mesh wire format: TreeSnapshot (crates/kv_index/src/snapshot.rs:18-52) and its producers / consumers
// (string_tree.rs:1066-1102 snapshot, :1228-1309 from_snapshot, :1318-1545 merge_snapshot).  bincode 1.3 default options:
// u64-LE lengths for Vec / String, fixed-width little-endian integers.
// =================================================================================================================
struct StringTreeIndex::SnapNode {
    std::string edge;                                        // UTF-8
    std::vector<std::pair<uint32_t, uint64_t>> tenants;      // (interned tenant, epoch), wire order
    std::vector<uint32_t> dup_tenants;                       // occurrences of a tenant beyond its first in the wire list (restore_node counts each)
    uint32_t child_count = 0;
    std::vector<std::pair<uint32_t, std::unique_ptr<SnapNode>>> kids;   // reconstructed remote tree: (first char, child), ascending
};

namespace {
void put64(std::string& b, uint64_t v) { for (int i = 0; i < 8; ++i) b.push_back((char)((v >> (8 * i)) & 0xFF)); }
bool get64(const uint8_t* b, size_t n, size_t& at, uint64_t& v) {
    if (n - at < 8) return false;
    v = 0;
    for (int i = 0; i < 8; ++i) v |= (uint64_t)b[at + i] << (8 * i);
    at += 8;
    return true;
}
}  // namespace

void StringTreeIndex::snapshot_bytes(std::string& out) const {
    out.clear();
    put64(out, 0);   // node count, patched below
    uint64_t count = 0;
    std::vector<uint32_t> stack{0};
    while (!stack.empty()) {   // pre-order, children ascending by char (children.sort_by_key, :1091)
        const uint32_t id = stack.back(); stack.pop_back();
        const Node& nd = nodes_[id];
        ++count;
        put64(out, nd.label_bytes);
        out.append((const char*)label(nd), nd.label_bytes);
        std::vector<std::pair<uint32_t, uint64_t>> ts(nd.tenants.begin(), nd.tenants.end());   // DashMap order is arbitrary: by name (DESIGN.md §3)
        std::sort(ts.begin(), ts.end(), [&](auto& a, auto& b) { return tenants_->rank[a.first] < tenants_->rank[b.first]; });
        put64(out, ts.size());
        for (auto& t : ts) { const std::string& name = tenants_->names[t.first]; put64(out, name.size()); out += name; put64(out, t.second); }
        const uint32_t cc = (uint32_t)nd.kids.size();
        for (int i = 0; i < 4; ++i) out.push_back((char)((cc >> (8 * i)) & 0xFF));
        for (size_t k = nd.kids.size(); k-- > 0;) stack.push_back(nd.kids[k].second);
    }
    for (int i = 0; i < 8; ++i) out[i] = (char)((count >> (8 * i)) & 0xFF);
}

// remote wins on a newer epoch; a tenant new to the node adds `chars` to its size (:1343-1369, :1392-1414, :1479-1500)
void StringTreeIndex::merge_tenant_list(uint32_t node, const std::vector<std::pair<uint32_t, uint64_t>>& remote, uint32_t chars) {
    bool changed = false;
    for (auto& kv : remote) {
        Node& nd = nodes_[node];
        const int64_t i = find_tenant(nd, kv.first);
        if (i < 0) { nd.tenants.emplace_back(kv.first, kv.second); tenant_chars_[kv.first] += chars; changed = true; }
        else if (kv.second > nd.tenants[(size_t)i].second) { nd.tenants[(size_t)i].second = kv.second; changed = true; }
    }
    if (changed) mark_node(node);
}

// clone_subtree / the trimmed remote node (:1422-1435, :1506-1520, :1563-1578) + accumulate_tenant_counts (:1548-1561): the remote
// node, its edge starting skip_bytes in, and everything below it become local nodes under `parent`
uint32_t StringTreeIndex::graft(uint32_t parent, const SnapNode& rn, size_t skip_bytes, bool count_dups) {
    const uint8_t* e = (const uint8_t*)rn.edge.data() + skip_bytes;
    const size_t nb = rn.edge.size() - skip_bytes;
    uint32_t cl;
    const uint32_t cp = utf8_first(e, &cl);
    const uint32_t chars = count_chars(e, nb);
    const uint64_t boff = bytes_.size();
    bytes_.insert(bytes_.end(), e, e + nb);
    const uint32_t id = new_node(boff, (uint32_t)nb, chars, parent, cp);
    for (auto& t : rn.tenants) { set_tenant(nodes_[id], t.first, t.second); tenant_chars_[t.first] += chars; }
    if (count_dups) for (uint32_t t : rn.dup_tenants) tenant_chars_[t] += chars;
    nodes_[id].last_tenant = -1;   // nodes restored from a snapshot carry no cached tenant (:1298-1304)
    const int64_t old = find_child(parent, cp);
    if (old >= 0) drop_subtree(table_[(size_t)old].child);   // DashMap::insert replaces
    table_insert(parent, cp, id);
    kids_insert(nodes_[parent], cp, id);
    for (auto& k : rn.kids) graft(id, *k.second, 0, count_dups);
    return id;
}

void StringTreeIndex::drop_subtree(uint32_t id) {
    const std::vector<std::pair<uint32_t, uint32_t>> kids = nodes_[id].kids;
    for (auto& k : kids) drop_subtree(k.second);
    table_erase(nodes_[id].parent, nodes_[id].first_cp);
    kids_erase(nodes_[nodes_[id].parent], nodes_[id].first_cp);
    free_node(id);
}

// merge_nodes(local, remote) (:1338-1545): only the remote node's tenants and children are read, never its edge
void StringTreeIndex::merge_nodes(uint32_t local, const SnapNode& remote) {
    merge_tenant_list(local, remote.tenants, nodes_[local].label_chars);
    for (auto& re : remote.kids) {
        const uint32_t rc = re.first;
        const SnapNode& rchild = *re.second;
        const int64_t slot = find_child(local, rc);
        if (slot < 0) { graft(local, rchild, 0); continue; }   // no local child at this char: the whole remote subtree (:1538-1543)
        const uint32_t m = table_[(size_t)slot].child;
        const size_t lb = nodes_[m].label_bytes, rb = rchild.edge.size();
        const size_t shared = shared_prefix_bytes((const uint8_t*)rchild.edge.data(), rb, label(nodes_[m]), lb);
        if (shared == lb && shared == rb) {            // case 1
            merge_nodes(m, rchild);
        } else if (shared == lb) {                     // case 2: the local edge is a prefix of the remote edge (:1385-1448)
            merge_tenant_list(m, rchild.tenants, nodes_[m].label_chars);
            uint32_t cl;
            const uint32_t rem_first = utf8_first((const uint8_t*)rchild.edge.data() + shared, &cl);
            const int64_t deeper = find_child(m, rem_first);
            if (deeper >= 0) merge_nodes(table_[(size_t)deeper].child, rchild);   // as in the reference: no edge comparison at this level
            else graft(m, rchild, shared);
        } else {                                       // case 3: split the local child at the shared prefix (:1449-1537)
            const uint32_t shared_chars = count_chars(label(nodes_[m]), shared);
            const uint64_t moff = nodes_[m].label_off;
            const uint32_t nn = new_node(moff, (uint32_t)shared, shared_chars, local, rc);
            nodes_[nn].tenants = nodes_[m].tenants;
            nodes_[nn].last_tenant = nodes_[m].last_tenant;
            nodes_[nn].split_epoch = nodes_[m].split_epoch = chunk_epoch_;
            Node& mm = nodes_[m];
            mm.label_off = moff + shared; mm.label_bytes -= (uint32_t)shared; mm.label_chars -= shared_chars; mm.parent = nn;
            uint32_t l2;
            mm.first_cp = utf8_first(label(mm), &l2);
            mark_node(m);
            kids_insert(nodes_[nn], mm.first_cp, m);
            table_set(local, rc, nn);
            kids_insert(nodes_[local], rc, nn);
            table_insert(nn, mm.first_cp, m);
            merge_tenant_list(nn, rchild.tenants, shared_chars);
            if (shared < rb) graft(nn, rchild, shared);   // a remote edge that IS the shared prefix loses its children (:1517)
        }
    }
}


// TreeSnapshot::from_bytes (snapshot.rs:49-51) = bincode::deserialize, i.e. bincode 1.3's DefaultOptions + fixint + allow_trailing_bytes:
// false = bincode error (short input, invalid UTF-8); bytes after the last node are accepted and ignored, as there
bool StringTreeIndex::decode_snapshot(const uint8_t* b, size_t n, std::vector<std::unique_ptr<SnapNode>>& flat) {
    size_t at = 0;
    uint64_t count;
    if (!get64(b, n, at, count)) return false;
    for (uint64_t i = 0; i < count; ++i) {
        auto nd = std::make_unique<SnapNode>();
        uint64_t len, nt;
        if (!get64(b, n, at, len) || n - at < len) return false;
        if (!valid_utf8(b + at, len)) return false;   // String deserialisation validates UTF-8
        nd->edge.assign((const char*)b + at, len); at += len;
        if (!get64(b, n, at, nt)) return false;
        for (uint64_t k = 0; k < nt; ++k) {
            uint64_t tl, ep;
            if (!get64(b, n, at, tl) || n - at < tl) return false;
            if (!valid_utf8(b + at, tl)) return false;
            const uint32_t t = tenants_->intern(std::string((const char*)b + at, tl)); at += tl;
            if (!get64(b, n, at, ep)) return false;
            bool seen = false;
            for (auto& kv : nd->tenants) if (kv.first == t) { kv.second = ep; seen = true; }   // DashMap::insert: the later entry wins
            if (seen) nd->dup_tenants.push_back(t); else nd->tenants.emplace_back(t, ep);
        }
        if (n - at < 4) return false;
        for (int k = 0; k < 4; ++k) nd->child_count |= (uint32_t)b[at + k] << (8 * k);
        at += 4;
        flat.push_back(std::move(nd));
    }
    return true;
}

// restore_node's shape (:1245-1309): pre-order list → tree; children with an empty edge are skipped with their subtrees, a later child
// with the same first char replaces an earlier one.  `lost` collects (tenant, chars) of everything restore_node would have counted in
// subtrees that end up replaced (from_snapshot keeps those counts).
std::unique_ptr<StringTreeIndex::SnapNode> StringTreeIndex::build_remote(std::vector<std::unique_ptr<SnapNode>>& flat, size_t& idx,
                                                                          std::vector<std::pair<uint32_t, uint32_t>>* lost) {
    std::unique_ptr<SnapNode> nd = std::move(flat[idx++]);
    for (uint32_t c = 0; c < nd->child_count; ++c) {
        if (idx >= flat.size()) break;
        if (flat[idx]->edge.empty()) {
            std::vector<size_t> todo{1};   // skip the node and all its descendants (:1284-1296)
            while (!todo.empty() && idx < flat.size()) {
                if (todo.back() == 0) { todo.pop_back(); continue; }
                --todo.back();
                todo.push_back(flat[idx++]->child_count);
            }
            continue;
        }
        std::unique_ptr<SnapNode> child = build_remote(flat, idx, lost);
        uint32_t cl;
        const uint32_t cp = utf8_first((const uint8_t*)child->edge.data(), &cl);
        auto it = std::lower_bound(nd->kids.begin(), nd->kids.end(), cp, [](auto& a, uint32_t v) { return a.first < v; });
        if (it != nd->kids.end() && it->first == cp) {
            if (lost) {
                std::vector<const SnapNode*> st{it->second.get()};
                while (!st.empty()) {
                    const SnapNode* x = st.back(); st.pop_back();
                    const uint32_t chars = count_chars((const uint8_t*)x->edge.data(), x->edge.size());
                    for (auto& t : x->tenants) lost->push_back({t.first, chars});
                    for (uint32_t t : x->dup_tenants) lost->push_back({t, chars});
                    for (auto& k : x->kids) st.push_back(k.second.get());
                }
            }
            it->second = std::move(child);
        } else nd->kids.insert(it, std::make_pair(cp, std::move(child)));
    }
    return nd;
}

bool StringTreeIndex::load_snapshot(const uint8_t* bytes, size_t n) {
    std::vector<std::unique_ptr<SnapNode>> flat;
    if (!decode_snapshot(bytes, n, flat)) return false;
    clear();
    if (flat.empty()) return true;
    size_t idx = 0;
    std::vector<std::pair<uint32_t, uint32_t>> lost;
    std::unique_ptr<SnapNode> root = build_remote(flat, idx, &lost);
    // the root: edge text (normally empty), tenants and their counts (:1258-1274)
    const uint32_t rchars = count_chars((const uint8_t*)root->edge.data(), root->edge.size());
    nodes_[0].label_off = bytes_.size();
    nodes_[0].label_bytes = (uint32_t)root->edge.size();
    nodes_[0].label_chars = rchars;
    bytes_.insert(bytes_.end(), root->edge.begin(), root->edge.end());
    for (auto& t : root->tenants) { set_tenant(nodes_[0], t.first, t.second); tenant_chars_[t.first] += rchars; }
    for (uint32_t t : root->dup_tenants) tenant_chars_[t] += rchars;
    for (auto& k : root->kids) graft(0, *k.second, 0, true);
    for (auto& l : lost) tenant_chars_[l.first] += l.second;
    mark_node(0);
    return true;
}

bool StringTreeIndex::merge_snapshot(const uint8_t* bytes, size_t n) {
    std::vector<std::unique_ptr<SnapNode>> flat;
    if (!decode_snapshot(bytes, n, flat)) return false;
    if (flat.empty()) return true;   // :1319-1321
    size_t idx = 0;
    std::unique_ptr<SnapNode> root = build_remote(flat, idx, nullptr);
    merge_nodes(0, *root);
    return true;
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

StrSlot StringTreeIndex::device_slot(uint32_t i) const {
    const StrChildSlot& c = table_[i];
    StrSlot t{c.key, c.child, 0, 0, 0, -1};
    if (c.key != 0 && c.child < kTombChild) {
        const Node& nd = nodes_[c.child];
        t.label_off = nd.label_off;
        t.label_bytes = nd.alive ? nd.label_bytes : 0;
        t.label_chars = (nd.alive ? nd.label_chars : 0) | (nd.alive && cache_valid(nd) ? kCacheValidBit : 0u);
        t.any_tenant = nd.alive ? any_tenant(nd) : -1;
    }
    return t;
}

StringTreeView StringTreeIndex::flush(cudaStream_t stream, uint64_t* launches) {
    if (!device_enabled) throw Error(SMGX_DEVICE_ERROR, "policy was created with device_id = -1 (host mirror only): no GPU path, no CPU fallback");
    if (tenants_version_seen != tenants_->version) { full_dirty_ = true; tenants_version_seen = tenants_->version; }
    // 32 B of slack past the arena: load16_global reads the aligned 16 B chunk after the one holding a label's last byte
    if (bytes_.size() + 32 > d_bytes_.cap) {
        if (stage_pending_) { SMGX_CUDA(cudaEventSynchronize(stage_done_)); stage_pending_ = false; }
        SMGX_CUDA(cudaDeviceSynchronize());
        d_bytes_.reserve(std::max<size_t>(bytes_.capacity() * 2, 4096) + 32);
        uploaded_bytes_ = 0;
    }
    if (uploaded_bytes_ < bytes_.size()) {
        SMGX_CUDA(cudaMemcpyAsync(d_bytes_.as<uint8_t>() + uploaded_bytes_, bytes_.data() + uploaded_bytes_, bytes_.size() - uploaded_bytes_,
                                  cudaMemcpyHostToDevice, stream));
        uploaded_bytes_ = bytes_.size();   // pageable source: the runtime has staged the bytes before the call returns
    }
    // a node whose header changed dirties the slot that points at it (the root has none: its state travels in the view)
    for (uint32_t id : dirty_nodes_) if (id < nodes_.size() && nodes_[id].slot != kNoNode) mark_slot(nodes_[id].slot);
    dirty_nodes_.clear();
    if (!full_dirty_ && dirty_slots_.size() > table_.size() / 8) full_dirty_ = true;
    if (full_dirty_) {
        if (stage_pending_) { SMGX_CUDA(cudaEventSynchronize(stage_done_)); stage_pending_ = false; }
        SMGX_CUDA(cudaDeviceSynchronize());
        std::vector<StrSlot> dev(table_.size());
        for (uint32_t i = 0; i < table_.size(); ++i) dev[i] = device_slot(i);
        d_table_.reserve(table_.size() * sizeof(StrSlot));
        SMGX_CUDA(cudaMemcpyAsync(d_table_.ptr, dev.data(), dev.size() * sizeof(StrSlot), cudaMemcpyHostToDevice, stream));
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
        for (size_t i = 0; i < ns; ++i) { const StrSlot t = device_slot(dirty_slots_[i]); memcpy(st + off_r + i * 32, &t, 32); }
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
    return StringTreeView{d_bytes_.as<uint8_t>(), d_table_.as<StrSlot>(), mask_, any_tenant(nodes_[0]), cache_valid(nodes_[0]) ? 1u : 0u};
}

// =================================================================================================================
// K2c + K3: longest char-aligned prefix walk + pick, one warp per request
// =================================================================================================================
namespace {
constexpr unsigned FULLM = 0xffffffffu;

// continuation bytes (10xxxxxx) in the 4 bytes of w
__device__ __forceinline__ uint32_t cont_bytes(uint32_t w) { return (uint32_t)__popc((w >> 7) & ~(w >> 6) & 0x01010101u); }

// 16 bytes starting at the arbitrarily aligned address `p`, from the two aligned 16-byte chunks around it.  The byte shift is the
// same for every lane of a warp whose addresses differ by multiples of 16, so the switch is warp-uniform.
__device__ __forceinline__ uint4 shift16(const uint4 lo, const uint4 hi, uint32_t s) {
    const uint32_t r = (s & 3) * 8;
    uint32_t w0, w1, w2, w3, w4;
    switch (s >> 2) {
        case 0: w0 = lo.x; w1 = lo.y; w2 = lo.z; w3 = lo.w; w4 = hi.x; break;
        case 1: w0 = lo.y; w1 = lo.z; w2 = lo.w; w3 = hi.x; w4 = hi.y; break;
        case 2: w0 = lo.z; w1 = lo.w; w2 = hi.x; w3 = hi.y; w4 = hi.z; break;
        default: w0 = lo.w; w1 = hi.x; w2 = hi.y; w3 = hi.z; w4 = hi.w; break;
    }
    return make_uint4(__funnelshift_r(w0, w1, r), __funnelshift_r(w1, w2, r), __funnelshift_r(w2, w3, r), __funnelshift_r(w3, w4, r));
}
__device__ __forceinline__ uint4 load16_global(const uint8_t* p) {
    const uint32_t s = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 15);
    const uint4* a = reinterpret_cast<const uint4*>(p - s);
    const uint4 lo = __ldg(a);
    if (s == 0) return lo;
    return shift16(lo, __ldg(a + 1), s);
}
// Both loads read the aligned 16-byte chunk holding p and, when p is unaligned, the next one: up to 30 bytes past p.  A lane whose
// 16 bytes start at a label's last byte therefore reads up to 30 bytes past the label's end — the label arena keeps 32 bytes of slack
// past its end (StringTreeIndex::flush), the staging window 32 bytes past kTxtWin.
__device__ __forceinline__ uint4 load16_shared(const uint8_t* p) {
    const uint32_t s = (uint32_t)(__cvta_generic_to_shared(p) & 15);
    const uint4* a = reinterpret_cast<const uint4*>(p - s);
    const uint4 lo = a[0];
    if (s == 0) return lo;
    return shift16(lo, a[1], s);
}

constexpr uint32_t kTxtWin = 4096;   // request bytes staged per warp (a whole chat-sized request)

// One warp per request.  The request is staged in shared memory 16 bytes per lane and load (char count taken on the way), labels
// are compared 512 bytes per step — 16 bytes per lane from the label (global, any alignment) against 16 from the staged request
// (shared, any alignment), both assembled from aligned 16-byte loads by a warp-uniform byte shift.
__global__ void __launch_bounds__(256) string_select_kernel(StringTreeView tv, FleetView f, const int32_t* __restrict__ slice_of_tenant,
                                                            const uint8_t* __restrict__ flags, uint32_t n_tenants, StringSelectArgs a) {
    __shared__ __align__(16) uint8_t win_all[8][kTxtWin + 32];
    const int lane = threadIdx.x & 31;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= a.count) return;
    const uint32_t r = a.first + w;
    const uint32_t off = a.offsets[r], nbytes = a.offsets[r + 1] - off;
    const uint8_t* s = a.text + off;
    uint8_t* win = win_all[threadIdx.x >> 5];
    uint32_t wbase = 0, wend = 0, wshift = 0;   // request bytes [wbase, wend) are staged; byte wbase sits at win[wshift]
    auto load_window = [&](uint32_t start) {
        __syncwarp();
        const uint8_t* g0 = s + start;
        wshift = (uint32_t)(reinterpret_cast<uintptr_t>(g0) & 15);
        wbase = start;
        wend = min(nbytes, start + kTxtWin - 16);
        const uint32_t span = wshift + (wend - wbase);                      // bytes to copy from the aligned address below g0
        const uint4* src = reinterpret_cast<const uint4*>(g0 - wshift);
        for (uint32_t c = lane; c * 16 < span; c += 32) reinterpret_cast<uint4*>(win)[c] = __ldg(src + c);   // only chunks that hold request bytes
        __syncwarp();
    };
    auto rq = [&](uint32_t pos) -> const uint8_t* { return win + wshift + (pos - wbase); };   // staged request byte `pos`
    // chars of the whole request = bytes − continuation bytes, streamed 16 bytes per lane (head / tail chunks byte by byte)
    uint32_t cont = 0;
    {
        const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(s) & 15);
        const uint4* src = reinterpret_cast<const uint4*>(s - sh);
        const uint32_t span = sh + nbytes;
        for (uint32_t c = lane; c * 16 < span; c += 32) {
            const uint4 v = __ldg(src + c);
            const uint32_t lo = c * 16, hi = lo + 16;
            if (lo >= sh && hi <= span) cont += cont_bytes(v.x) + cont_bytes(v.y) + cont_bytes(v.z) + cont_bytes(v.w);
            else {
                const uint32_t ws[4] = {v.x, v.y, v.z, v.w};
                for (uint32_t k = 0; k < 16; ++k) { const uint32_t g = lo + k; if (g >= sh && g < span) cont += (((ws[k >> 2] >> (8 * (k & 3))) & 0xC0) == 0x80); }
            }
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) cont += __shfl_xor_sync(FULLM, cont, d);
    }
    const uint32_t input_chars = nbytes - cont;
    if (nbytes) load_window(0);

    uint32_t cur = 0, pos = 0, matched = 0, terminal = 0, visited = 0;
    int32_t term_tenant = tv.root_tenant;       // tenant / cache flag of the node the walk currently ends on
    uint32_t term_cache = tv.root_cache_valid;
    while (pos < nbytes) {
        if (pos < wbase || pos + 4 > wend) { if (!(pos >= wbase && wend == nbytes)) load_window(pos); }
        uint32_t cl;
        const uint32_t cp = utf8_first(rq(pos), &cl);   // every lane reads the same ≤ 4 staged bytes
        const uint64_t key = str_child_key(cur, cp);
        uint32_t idx = str_child_home(key) & tv.child_mask;
        uint32_t child = kNoNode;
        uint4 s4, h4{};
        for (;;) {   // warp-uniform probe; a hit carries the child's header in the same 32 B
            const uint4* sp = reinterpret_cast<const uint4*>(tv.slots + idx);
            s4 = __ldg(sp);
            const uint64_t skey = ((uint64_t)s4.y << 32) | s4.x;
            if (skey == 0) break;
            if (skey == key && s4.z < kTombChild) { child = s4.z; h4 = __ldg(sp + 1); break; }
            idx = (idx + 1) & tv.child_mask;
        }
        if (child == kNoNode) break;
        const uint64_t label_off = ((uint64_t)h4.y << 32) | h4.x;
        const uint32_t label_bytes = s4.w, label_chars = h4.z & ~kCacheValidBit;
        term_tenant = (int32_t)h4.w;
        term_cache = (h4.z & kCacheValidBit) ? 1u : 0u;
        const uint8_t* lab = tv.bytes + label_off;
        const uint32_t L = min(label_bytes, nbytes - pos);
        uint32_t common = L;
        for (uint32_t c = 0; c < L; c += 512) {
            if (pos + c < wbase || pos + c + min(512u, L - c) > wend) load_window(pos + c);
            const uint32_t b = c + (uint32_t)lane * 16;
            uint32_t first = 16;   // index of my first differing byte
            if (b < L) {
                const uint4 x = load16_global(lab + b), y = load16_shared(rq(pos + b));
                const uint32_t nv = min(16u, L - b);
                const uint32_t dw[4] = {x.x ^ y.x, x.y ^ y.y, x.z ^ y.z, x.w ^ y.w};
#pragma unroll
                for (int k = 3; k >= 0; --k) if (dw[k]) first = (uint32_t)k * 4 + ((uint32_t)__ffs((int)dw[k]) - 1) / 8;
                if (first >= nv) first = 16;
            }
            const unsigned mm = __ballot_sync(FULLM, first < 16);
            if (mm) {
                const int src = __ffs((int)mm) - 1;
                common = c + (uint32_t)src * 16 + __shfl_sync(FULLM, first, src);
                break;
            }
        }
        if (common < L) {   // mismatch inside a char: back to its first byte (at most 3 bytes back)
            const uint32_t back = min(common, 4u);
            if (pos + common - back < wbase || pos + common >= wend) load_window(pos + common - back);
            while (common > 0 && (*rq(pos + common) & 0xC0) == 0x80) --common;
        }
        uint32_t shared_chars = label_chars;
        if (common != label_bytes) {   // chars in the matched part of the edge
            uint32_t cb = 0;
            for (uint32_t c0 = 0; c0 < common; c0 += 2048) {
                const uint32_t c1 = min(common, c0 + 2048);
                if (pos + c0 < wbase || pos + c1 > wend) load_window(pos + c0);
                for (uint32_t i = c0 + lane; i < c1; i += 32) cb += (*rq(pos + i) & 0xC0) == 0x80;
            }
#pragma unroll
            for (int d = 16; d; d >>= 1) cb += __shfl_xor_sync(FULLM, cb, d);
            shared_chars = common - cb;
        }
        matched += shared_chars;
        terminal = child;                       // a partial edge match still selects that child (:582-586)
        ++visited;
        if (common != label_bytes) break;
        pos += common;
        cur = child;
    }
    if (lane != 0) return;
    const int32_t tenant = term_tenant;
    a.out_node[r] = terminal;
    a.out_tenant[r] = tenant;
    a.out_fill[r] = term_cache ? 0 : 1;
    int32_t out = -1;
    uint32_t branch = SMGX_BR_NO_HEALTHY;
    if (a.decide) {
        const FleetDerived fd = *f.derived;
        if (fd.n_healthy == 0) {
        } else if (fd.imbalanced) {
            out = fd.min_load_idx; branch = SMGX_BR_IMBALANCED_MIN_LOAD;
        } else {
            // match_rate = matched_char_count as f32 / input_char_count as f32, 0 chars → 0.0, strict > (cache_aware.rs:917-927)
            const float rate = input_chars == 0 ? 0.0f : __fdiv_rn(__uint2float_rn(matched), __uint2float_rn(input_chars));
            if (rate > a.cache_threshold) {
                const int32_t sl = (tenant >= 0 && (uint32_t)tenant < n_tenants) ? slice_of_tenant[tenant] : -1;
                if (sl >= 0 && (flags[sl] & 1)) { out = sl; branch = SMGX_BR_TREE_MATCH; }
                else { out = fd.first_healthy; branch = SMGX_BR_TREE_FALLBACK_FIRST_HEALTHY; }
            } else { out = fd.min_load_idx; branch = SMGX_BR_TREE_MIN_LOAD; }
        }
    }
    a.out_idx[r] = out;
    if (a.out_info) {
        smgx_decision_info di;
        di.matched = matched; di.input = input_chars; di.branch = (uint8_t)branch;
        di.nodes = (uint8_t)min(visited, 255u); di.reserved[0] = di.reserved[1] = 0;
        a.out_info[r] = di;
    }
}
}  // namespace

void launch_string_select(const StringTreeView& tv, const FleetView& fleet, const int32_t* d_slice_of_tenant, const uint8_t* d_flags,
                          uint32_t n_tenants, const StringSelectArgs& a, cudaStream_t stream) {
    if (a.count == 0) return;
    string_select_kernel<<<(unsigned)(((uint64_t)a.count * 32 + 255) / 256), 256, 0, stream>>>(tv, fleet, d_slice_of_tenant, d_flags, n_tenants, a);
    SMGX_CUDA(cudaGetLastError());
}

}  // namespace smgx
