// Host-side writer + device mirror of the positional KV index.  See event_index.h for the layout and the
// reference functions each method replaces (crates/kv_index/src/event_tree.rs).
#include "event_index.h"

#include <algorithm>
#include <cstring>

#include "xxh3.cuh"

namespace smgx {

namespace {

// 32-byte records (Slot / MultiNode / RunRec): two threads per record, 16 B each → coalesced 32 B sector writes.  Records n1.. go to
// dst2 instead of dst (the slots' records, in the same launch as the slots).  For slots (tags != nullptr) the thread that writes the
// first half (content, pos, state) writes the slot's tag as well.
__global__ void scatter32_kernel(uint4* __restrict__ dst, const uint32_t* __restrict__ idx, const uint4* __restrict__ src,
                                 uint32_t n, uint8_t* __restrict__ tags, uint4* __restrict__ dst2, uint32_t n1) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t rec = t >> 1, half = t & 1;
    if (rec >= n) return;
    const uint32_t i = idx[rec];
    const uint4 r = src[(size_t)rec * 2 + half];
    if (rec >= n1) { dst2[(size_t)i * 2 + half] = r; return; }
    dst[(size_t)i * 2 + half] = r;
    if (tags && half == 0) tags[i] = slot_tag(r.w, r.z, (uint64_t)r.x | ((uint64_t)r.y << 32));
}
// every tag from the slots after a bulk upload; one thread per 4 slots writes one u32 of tags
__global__ void derive_tags_kernel(const uint4* __restrict__ slots, uint32_t* __restrict__ tags, uint32_t n4) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n4) return;
    uint32_t w = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint4 r = slots[((size_t)t * 4 + k) * 2];
        w |= (uint32_t)slot_tag(r.w, r.z, (uint64_t)r.x | ((uint64_t)r.y << 32)) << (8 * k);
    }
    tags[t] = w;
}
__global__ void scatter_rows_kernel(uint64_t* __restrict__ dst, const uint32_t* __restrict__ idx, const uint64_t* __restrict__ src,
                                    uint32_t n, uint32_t words) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t rec = t / words, w = t % words;
    if (rec < n) dst[(size_t)idx[rec] * words + w] = src[(size_t)rec * words + w];
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

EventIndex::EventIndex(uint32_t jump_size) : jump_(jump_size) {
    if (jump_size == 0) throw Error(SMGX_INVALID_ARGUMENT, "jump_size must be greater than 0");  // event_tree.rs:280
    slots_.assign(1024, Slot{0, 0, SLOT_EMPTY, kNil, 0, 0});
    prefix_.assign(1024, 0);
    mask_ = 1023;
}

EventIndex::~EventIndex() {
    d_slots_.release(); d_rows_.release(); d_multi_.release(); d_tree_.release(); d_tags_.release(); d_runs_.release(); d_stage_.release(); stage_.release();
    if (stage_done_) cudaEventDestroy(stage_done_);
}

// ---------------------------------------------------------------------------------------------------------------
// worker interning (event_tree.rs:509-525)
// ---------------------------------------------------------------------------------------------------------------
uint32_t EventIndex::intern_worker(const std::string& url) {
    auto it = worker_to_id_.find(url);
    if (it != worker_to_id_.end()) return it->second;
    uint32_t id = (uint32_t)tree_sizes_.size();
    if (id >= kMaxWords * 64)
        throw Error(SMGX_INVALID_ARGUMENT, "worker count " + std::to_string(id) + " exceeds MAX_WORKERS (2048) per device shard");
    if (id >= words_ * 64) {
        uint32_t nw = words_;
        while (id >= nw * 64) nw *= 2;
        rebuild((uint32_t)slots_.size(), nw);
    }
    worker_to_id_[url] = id;
    tree_sizes_.push_back(0);
    worker_blocks_.emplace_back();
    tree_dirty_ = true;
    ++workers_version_;
    return id;
}

int64_t EventIndex::worker_id(const std::string& url) const {
    auto it = worker_to_id_.find(url);
    return it == worker_to_id_.end() ? -1 : (int64_t)it->second;
}

uint64_t EventIndex::current_size() const {
    uint64_t s = 0;
    for (uint64_t v : tree_sizes_) s += v;
    return s;
}

// ---------------------------------------------------------------------------------------------------------------
// worker bitsets
// ---------------------------------------------------------------------------------------------------------------
uint64_t* EventIndex::set_words(uint64_t& payload) { return words_ == 1 ? &payload : &rows_[(size_t)payload * words_]; }

uint64_t EventIndex::new_set(uint32_t wid) {
    if (words_ == 1) return 1ULL << wid;
    uint32_t row;
    if (!free_rows_.empty()) { row = free_rows_.back(); free_rows_.pop_back(); }
    else {
        row = (uint32_t)(rows_.size() / words_);
        size_t before = rows_.capacity();
        rows_.resize(rows_.size() + words_, 0);
        if (rows_.capacity() != before) full_dirty_ = true;  // device array must be re-sized as well
    }
    std::fill(rows_.begin() + (size_t)row * words_, rows_.begin() + (size_t)(row + 1) * words_, 0ULL);
    rows_[(size_t)row * words_ + (wid >> 6)] = 1ULL << (wid & 63);
    mark_row(row);
    return row;
}
void EventIndex::free_set(uint64_t payload) { if (words_ > 1) free_rows_.push_back((uint32_t)payload); }
bool EventIndex::set_empty(uint64_t& payload) {
    uint64_t* w = set_words(payload);
    for (uint32_t i = 0; i < words_; ++i) if (w[i]) return false;
    return true;
}
void EventIndex::mark_set_dirty(uint64_t payload) { if (words_ > 1) mark_row((uint32_t)payload); }

// ---------------------------------------------------------------------------------------------------------------
// open-addressed table on the host mirror
// ---------------------------------------------------------------------------------------------------------------
int64_t EventIndex::find_slot(uint32_t pos, uint64_t content) const {
    uint32_t h = slot_hash(pos, content) & mask_;
    for (;;) {
        const Slot& s = slots_[h];
        if (s.state == SLOT_EMPTY) return -1;
        if (s.state != SLOT_TOMB && s.content == content && s.pos == pos) return h;
        h = (h + 1) & mask_;
    }
}

// Claims a slot for a key known to be absent (re-uses the first tombstone on the probe path).
uint32_t EventIndex::insert_slot(uint32_t pos, uint64_t content) {
    if ((live_ + tombs_ + 1) * 2 > slots_.size()) {
        uint32_t cap = (uint32_t)slots_.size();
        while ((live_ + 1) * 4 > cap) cap *= 2;   // ≤ 25 % live after a rebuild
        rebuild(cap, words_);
    }
    uint32_t h = slot_hash(pos, content) & mask_;
    int64_t tomb = -1;
    for (;;) {
        Slot& s = slots_[h];
        if (s.state == SLOT_EMPTY) break;
        if (s.state == SLOT_TOMB && tomb < 0) tomb = h;
        h = (h + 1) & mask_;
    }
    if (tomb >= 0) { h = (uint32_t)tomb; --tombs_; }
    ++live_;
    slots_[h].content = content;
    slots_[h].pos = pos;
    return h;
}

uint32_t EventIndex::new_multi(uint64_t prefix, uint64_t payload, uint32_t next) {
    uint32_t i;
    if (!free_multi_.empty()) { i = free_multi_.back(); free_multi_.pop_back(); }
    else {
        i = (uint32_t)multi_.size();
        size_t before = multi_.capacity();
        multi_.push_back(MultiNode{});
        if (multi_.capacity() != before) full_dirty_ = true;
    }
    multi_[i] = MultiNode{prefix, payload, next, 0, 0};
    mark_multi(i);
    return i;
}

// SeqEntry::new / SeqEntry::insert (event_tree.rs:170-192) behind DashMap::entry().and_modify().or_insert_with() (:344-347)
// A new key takes record `i` of the run being written (the last one); an existing key keeps the record it has.
void EventIndex::insert_entry(uint32_t pos, uint64_t content, uint64_t prefix, uint32_t wid, uint32_t i) {
    int64_t f = find_slot(pos, content);
    if (f < 0) {
        uint32_t h = insert_slot(pos, content);   // a rebuild in there may move the run, never split it
        Slot& s = slots_[h];
        s.state = SLOT_SINGLE;
        s.run = run_starts_.back() + i;
        prefix_[h] = prefix;
        s.payload = new_set(wid);
        mark_slot(h);
        return;
    }
    Slot& s = slots_[(size_t)f];
    if (s.state == SLOT_SINGLE) {
        if (prefix_[(size_t)f] == prefix) {
            uint64_t* w = set_words(s.payload);
            w[wid >> 6] |= 1ULL << (wid & 63);
            if (words_ == 1) mark_slot((uint32_t)f); else mark_set_dirty(s.payload);
            return;
        }
        // Single → Multi upgrade; never downgrades (:182-187)
        uint32_t a = new_multi(prefix_[(size_t)f], s.payload, kNil);
        uint64_t nset = new_set(wid);
        uint32_t b = new_multi(prefix, nset, a);
        Slot& s2 = slots_[(size_t)f];  // new_set may have grown rows_, never slots_
        s2.state = SLOT_MULTI;
        ++multi_slots_;
        prefix_[(size_t)f] = 0;
        s2.payload = b;
        mark_slot((uint32_t)f);
        return;
    }
    // Multi: map.entry(seq_hash).or_default().insert(worker) (:188-190)
    for (uint32_t i = (uint32_t)s.payload; i != kNil; i = multi_[i].next) {
        if (multi_[i].prefix == prefix) {
            uint64_t* w = set_words(multi_[i].payload);
            w[wid >> 6] |= 1ULL << (wid & 63);
            if (words_ == 1) mark_multi(i); else mark_set_dirty(multi_[i].payload);
            return;
        }
    }
    uint64_t nset = new_set(wid);
    uint32_t head = new_multi(prefix, nset, (uint32_t)slots_[(size_t)f].payload);
    slots_[(size_t)f].payload = head;
    mark_slot((uint32_t)f);
}

// SeqEntry::remove + Entry::Occupied::remove when empty (event_tree.rs:196-213, :393-397)
void EventIndex::drop_entry(const BlockRec& r, uint32_t wid) {
    int64_t f = find_slot(r.pos, r.content);
    if (f < 0) return;
    Slot& s = slots_[(size_t)f];
    bool now_empty = false;
    if (s.state == SLOT_SINGLE) {
        if (prefix_[(size_t)f] != r.prefix) return;
        uint64_t* w = set_words(s.payload);
        w[wid >> 6] &= ~(1ULL << (wid & 63));
        if (set_empty(s.payload)) { free_set(s.payload); now_empty = true; }
        else if (words_ > 1) mark_set_dirty(s.payload);
    } else {
        uint32_t prev = kNil;
        for (uint32_t i = (uint32_t)s.payload; i != kNil; prev = i, i = multi_[i].next) {
            if (multi_[i].prefix != r.prefix) continue;
            uint64_t* w = set_words(multi_[i].payload);
            w[wid >> 6] &= ~(1ULL << (wid & 63));
            if (set_empty(multi_[i].payload)) {
                free_set(multi_[i].payload);
                uint32_t nx = multi_[i].next;
                if (prev == kNil) s.payload = nx; else { multi_[prev].next = nx; mark_multi(prev); }
                free_multi_.push_back(i);
            } else if (words_ == 1) mark_multi(i); else mark_set_dirty(multi_[i].payload);
            break;
        }
        now_empty = (uint32_t)s.payload == kNil;
    }
    if (now_empty) {
        if (s.state == SLOT_MULTI) --multi_slots_;
        s.state = SLOT_TOMB;
        s.payload = 0;
        --live_;
        ++tombs_;
    }
    mark_slot((uint32_t)f);   // a tombstone's record goes dead, and the slot lets go of it
    if (now_empty) s.run = kNil;
}

// ---------------------------------------------------------------------------------------------------------------
// events (event_tree.rs:305-435)
// ---------------------------------------------------------------------------------------------------------------
smgx_status EventIndex::apply_stored(uint32_t wid, const uint64_t* seq, const uint64_t* content, uint32_t n, const uint64_t* parent) {
    if (wid >= tree_sizes_.size()) throw Error(SMGX_INVALID_ARGUMENT, "unknown worker id");
    if (n == 0) return SMGX_SUCCESS;
    auto& wb = worker_blocks_[wid];
    uint32_t start = 0;
    bool have_prev = false;
    uint64_t prev = 0;
    if (parent) {
        if (wb.empty()) return SMGX_WORKER_NOT_TRACKED;
        auto it = wb.find(*parent);
        if (it == wb.end()) return SMGX_PARENT_BLOCK_NOT_FOUND;
        start = it->second.pos + 1;
        prev = it->second.prefix;
        have_prev = true;
    }
    // compact when dead records outnumber live entries, and not before the arena has doubled since the last compaction: runs
    // that each keep one live record cannot shrink, and must not make every call pay for a pass over the arena
    if (runs_.size() - live_ > std::max<uint64_t>(live_, 1024) && runs_.size() >= 2 * runs_kept_) compact_runs();
    if (runs_.size() + n > kNil) throw Error(SMGX_INVALID_ARGUMENT, "event index run arena exceeds 2^32 - 1 records");
    // one run of n records, position order; a record stays dead unless its block creates a key
    const size_t before = runs_.capacity();
    run_starts_.push_back((uint32_t)runs_.size());
    runs_.resize(runs_.size() + n, RunRec{0, 0, SLOT_EMPTY, 0, 0});
    if (runs_.capacity() != before) full_dirty_ = true;   // device array must be re-sized as well
    // the dead records are not uploaded: the device array is zero (dead) past the end of the last full upload
    uint64_t fresh = 0;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t pos = start + i;
        uint64_t c = content[i];
        uint64_t pfx = have_prev ? xxh3_pair(prev, c, kSeed) : c;  // :338-342
        insert_entry(pos, c, pfx, wid, i);
        auto ins = wb.insert_or_assign(seq[i], BlockRec{pos, c, pfx});
        if (ins.second) ++fresh;  // only genuinely new seq hashes count (:349-356)
        prev = pfx;
        have_prev = true;
    }
    if (fresh) { tree_sizes_[wid] += fresh; tree_dirty_ = true; }
    return SMGX_SUCCESS;
}

void EventIndex::apply_removed(uint32_t wid, const uint64_t* seq, uint32_t n) {
    if (wid >= tree_sizes_.size()) throw Error(SMGX_INVALID_ARGUMENT, "unknown worker id");
    auto& wb = worker_blocks_[wid];
    uint64_t removed = 0;
    for (uint32_t i = 0; i < n; ++i) {
        auto it = wb.find(seq[i]);
        if (it == wb.end()) continue;
        BlockRec r = it->second;
        wb.erase(it);
        drop_entry(r, wid);
        ++removed;
    }
    if (removed) { tree_sizes_[wid] -= removed; tree_dirty_ = true; }
}

void EventIndex::apply_cleared(uint32_t wid) {
    if (wid >= tree_sizes_.size()) throw Error(SMGX_INVALID_ARGUMENT, "unknown worker id");
    auto& wb = worker_blocks_[wid];
    for (auto& kv : wb) drop_entry(kv.second, wid);
    wb.clear();
    tree_sizes_[wid] = 0;
    tree_dirty_ = true;
}

void EventIndex::remove_worker(uint32_t wid) { apply_cleared(wid); }

// ---------------------------------------------------------------------------------------------------------------
// rebuild (growth of the table or of the bitset width) — re-lays out everything, then a bulk upload
// ---------------------------------------------------------------------------------------------------------------
void EventIndex::rebuild(uint32_t new_capacity, uint32_t new_words) {
    std::vector<Slot> old_slots;
    old_slots.swap(slots_);
    std::vector<uint64_t> old_prefix;
    old_prefix.swap(prefix_);
    std::vector<uint64_t> old_rows;
    old_rows.swap(rows_);
    std::vector<MultiNode> old_multi;
    old_multi.swap(multi_);
    uint32_t old_words = words_;
    free_rows_.clear();
    free_multi_.clear();
    words_ = new_words;
    slots_.assign(new_capacity, Slot{0, 0, SLOT_EMPTY, kNil, 0, 0});
    prefix_.assign(new_capacity, 0);
    mask_ = new_capacity - 1;
    live_ = 0;
    tombs_ = 0;
    multi_slots_ = 0;
    full_dirty_ = true;
    dirty_slots_.clear(); dirty_multi_.clear(); dirty_rows_.clear(); dirty_runs_.clear();

    auto convert = [&](uint64_t old_payload) -> uint64_t {
        const uint64_t* src = old_words == 1 ? &old_payload : &old_rows[(size_t)old_payload * old_words];
        if (new_words == 1) return src[0];
        uint32_t row = (uint32_t)(rows_.size() / new_words);
        rows_.resize(rows_.size() + new_words, 0);
        for (uint32_t i = 0; i < old_words && i < new_words; ++i) rows_[(size_t)row * new_words + i] = src[i];
        return row;
    };
    for (size_t oi = 0; oi < old_slots.size(); ++oi) {
        const Slot& o = old_slots[oi];
        if (o.state != SLOT_SINGLE && o.state != SLOT_MULTI) continue;
        uint32_t h = slot_hash(o.pos, o.content) & mask_;
        while (slots_[h].state != SLOT_EMPTY) h = (h + 1) & mask_;
        ++live_;
        Slot& s = slots_[h];
        s.content = o.content; s.pos = o.pos; s.state = o.state; s.run = o.run;
        prefix_[h] = old_prefix[oi];
        if (o.state == SLOT_SINGLE) s.payload = convert(o.payload);
        else {
            ++multi_slots_;
            uint32_t head = kNil;
            for (uint32_t i = (uint32_t)o.payload; i != kNil; i = old_multi[i].next) {
                uint32_t ni = (uint32_t)multi_.size();
                multi_.push_back(MultiNode{old_multi[i].prefix, convert(old_multi[i].payload), head, 0, 0});
                head = ni;
            }
            s.payload = head;
        }
        mark_slot(h);   // the record takes the converted payload
    }
    compact_runs();
}

// Drops the runs that hold no live record and closes the gaps; records never move inside a run, so anchor + position stays
// the layout of every run kept.  The last run is always kept: a rebuild in the middle of apply_stored compacts while that
// call is still filling it.  The slots' `run` indices are remapped; the whole index is uploaded again.
void EventIndex::compact_runs() {
    std::vector<uint32_t> remap(runs_.size(), kNil);
    std::vector<uint32_t> starts;
    uint32_t out = 0;
    for (size_t k = 0; k < run_starts_.size(); ++k) {
        const uint32_t b = run_starts_[k], e = k + 1 < run_starts_.size() ? run_starts_[k + 1] : (uint32_t)runs_.size();
        bool live = k + 1 == run_starts_.size();
        for (uint32_t i = b; i < e && !live; ++i) live = runs_[i].state != SLOT_EMPTY;
        if (!live) continue;
        starts.push_back(out);
        for (uint32_t i = b; i < e; ++i) { remap[i] = out; runs_[out++] = runs_[i]; }
    }
    runs_.resize(out);
    runs_kept_ = out;
    run_starts_.swap(starts);
    for (Slot& s : slots_)
        if (s.run != kNil) s.run = remap[s.run];
    full_dirty_ = true;
    dirty_slots_.clear(); dirty_multi_.clear(); dirty_rows_.clear(); dirty_runs_.clear();
}

// ---------------------------------------------------------------------------------------------------------------
// device mirror
// ---------------------------------------------------------------------------------------------------------------
EventIndexView EventIndex::flush(cudaStream_t stream, uint64_t* launches) {
    if (!device_enabled) throw Error(SMGX_DEVICE_ERROR, "policy was created with device_id = -1 (host mirror only): no GPU path, no CPU fallback");
    size_t n_dirty = dirty_slots_.size() + dirty_multi_.size() + dirty_rows_.size();   // a dirty record comes with its dirty slot
    if (!full_dirty_ && n_dirty > slots_.size() / 8) full_dirty_ = true;
    if (full_dirty_) {
        if (stage_pending_) { SMGX_CUDA(cudaEventSynchronize(stage_done_)); stage_pending_ = false; }
        // growth re-allocates: make sure no kernel still reads the old arrays
        SMGX_CUDA(cudaDeviceSynchronize());
        d_slots_.reserve(slots_.size() * sizeof(Slot));
        d_rows_.reserve(std::max<size_t>(rows_.capacity(), 1) * sizeof(uint64_t));
        d_multi_.reserve(std::max<size_t>(multi_.capacity(), 1) * sizeof(MultiNode));
        d_tags_.reserve(slots_.size());
        d_runs_.reserve(std::max<size_t>(runs_.capacity(), 1) * sizeof(RunRec));
        SMGX_CUDA(cudaMemcpyAsync(d_slots_.ptr, slots_.data(), slots_.size() * sizeof(Slot), cudaMemcpyHostToDevice, stream));
        const uint32_t n4 = (uint32_t)(slots_.size() / 4);   // capacity: a power of two ≥ 1024
        derive_tags_kernel<<<(n4 + 255) / 256, 256, 0, stream>>>(d_slots_.as<uint4>(), d_tags_.as<uint32_t>(), n4);
        SMGX_CUDA(cudaGetLastError());
        ++*launches;
        if (!rows_.empty())
            SMGX_CUDA(cudaMemcpyAsync(d_rows_.ptr, rows_.data(), rows_.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, stream));
        if (!multi_.empty())
            SMGX_CUDA(cudaMemcpyAsync(d_multi_.ptr, multi_.data(), multi_.size() * sizeof(MultiNode), cudaMemcpyHostToDevice, stream));
        if (!runs_.empty())
            SMGX_CUDA(cudaMemcpyAsync(d_runs_.ptr, runs_.data(), runs_.size() * sizeof(RunRec), cudaMemcpyHostToDevice, stream));
        // records appended later are uploaded only where a key makes them live: the rest must read as dead, not as what a
        // compaction left there
        SMGX_CUDA(cudaMemsetAsync(d_runs_.as<char>() + runs_.size() * sizeof(RunRec), 0, d_runs_.cap - runs_.size() * sizeof(RunRec), stream));
        full_dirty_ = false;
        dirty_slots_.clear(); dirty_multi_.clear(); dirty_rows_.clear(); dirty_runs_.clear();
        tree_dirty_ = true;
    } else if (n_dirty) {
        if (!stage_done_) SMGX_CUDA(cudaEventCreateWithFlags(&stage_done_, cudaEventDisableTiming));
        if (stage_pending_) { SMGX_CUDA(cudaEventSynchronize(stage_done_)); stage_pending_ = false; }
        auto uniq = [](std::vector<uint32_t>& v) { std::sort(v.begin(), v.end()); v.erase(std::unique(v.begin(), v.end()), v.end()); };
        uniq(dirty_slots_); uniq(dirty_multi_); uniq(dirty_rows_); uniq(dirty_runs_);
        size_t ns = dirty_slots_.size(), nm = dirty_multi_.size(), nr = dirty_rows_.size(), nu = dirty_runs_.size();
        // staging layout: [slot idx][run idx][multi idx][row idx] | 32B-aligned [slot recs][run recs][multi recs][row words]
        size_t off_si = 0, off_ui = off_si + ns * 4, off_mi = off_ui + nu * 4, off_ri = off_mi + nm * 4;
        size_t off_sr = align_up(off_ri + nr * 4, 32), off_ur = off_sr + ns * 32, off_mr = off_ur + nu * 32, off_rr = off_mr + nm * 32;
        size_t total = off_rr + nr * words_ * 8;
        stage_.reserve(total);
        d_stage_.reserve(total);
        char* st = stage_.as<char>();
        memcpy(st + off_si, dirty_slots_.data(), ns * 4);
        memcpy(st + off_mi, dirty_multi_.data(), nm * 4);
        memcpy(st + off_ui, dirty_runs_.data(), nu * 4);
        memcpy(st + off_ri, dirty_rows_.data(), nr * 4);
        for (size_t i = 0; i < ns; ++i) memcpy(st + off_sr + i * 32, &slots_[dirty_slots_[i]], 32);
        for (size_t i = 0; i < nm; ++i) memcpy(st + off_mr + i * 32, &multi_[dirty_multi_[i]], 32);
        for (size_t i = 0; i < nu; ++i) memcpy(st + off_ur + i * 32, &runs_[dirty_runs_[i]], 32);
        for (size_t i = 0; i < nr; ++i) memcpy(st + off_rr + i * words_ * 8, &rows_[(size_t)dirty_rows_[i] * words_], words_ * 8);
        SMGX_CUDA(cudaMemcpyAsync(d_stage_.ptr, st, total, cudaMemcpyHostToDevice, stream));
        char* ds = d_stage_.as<char>();
        if (ns + nu) {   // a record is dirty only with its slot: the slots and their records in one launch
            scatter32_kernel<<<(unsigned)(((ns + nu) * 2 + 255) / 256), 256, 0, stream>>>(
                d_slots_.as<uint4>(), (const uint32_t*)(ds + off_si), (const uint4*)(ds + off_sr), (uint32_t)(ns + nu), d_tags_.as<uint8_t>(),
                d_runs_.as<uint4>(), (uint32_t)ns);
            ++*launches;
        }
        if (nm) {
            scatter32_kernel<<<(unsigned)((nm * 2 + 255) / 256), 256, 0, stream>>>(d_multi_.as<uint4>(), (const uint32_t*)(ds + off_mi),
                                                                                 (const uint4*)(ds + off_mr), (uint32_t)nm, nullptr, nullptr, (uint32_t)nm);
            ++*launches;
        }
        if (nr) {
            scatter_rows_kernel<<<(unsigned)((nr * words_ + 255) / 256), 256, 0, stream>>>(
                d_rows_.as<uint64_t>(), (const uint32_t*)(ds + off_ri), (const uint64_t*)(ds + off_rr), (uint32_t)nr, words_);
            ++*launches;
        }
        SMGX_CUDA(cudaGetLastError());
        SMGX_CUDA(cudaEventRecord(stage_done_, stream));
        stage_pending_ = true;
        dirty_slots_.clear(); dirty_multi_.clear(); dirty_rows_.clear(); dirty_runs_.clear();
    }
    if (tree_dirty_) {
        d_tree_.reserve(std::max<size_t>(tree_sizes_.size(), 1) * 8);
        if (!tree_sizes_.empty())
            SMGX_CUDA(cudaMemcpyAsync(d_tree_.ptr, tree_sizes_.data(), tree_sizes_.size() * 8, cudaMemcpyHostToDevice, stream));
        tree_dirty_ = false;
    }
    EventIndexView v;
    v.slots = d_slots_.as<Slot>();
    v.rows = d_rows_.as<uint64_t>();
    v.multi = d_multi_.as<MultiNode>();
    v.tree_sizes = d_tree_.as<uint64_t>();
    v.tags = d_tags_.as<uint8_t>();
    v.runs = d_runs_.as<RunRec>();
    v.n_runs = (uint32_t)runs_.size();
    v.mask = mask_;
    v.words = words_;
    v.n_workers = (uint32_t)tree_sizes_.size();
    v.jump = jump_;
    return v;
}

}  // namespace smgx
