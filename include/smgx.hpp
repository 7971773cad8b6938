// smgx.hpp — C++17 host mirror of the reference's plugin interface for the cache_aware path, over the C ABI (smgx.h).
//
// The reference is Rust; its toolchain is absent from this image, so the host side above the C ABI is written in C++ with the
// reference's names, argument meaning and error behaviour (Python twin for the test-suite: smg_b200/policy.py):
//   trait LoadBalancingPolicy          model_gateway/src/policies/mod.rs:43-86      → smgx::LoadBalancingPolicy
//   struct CacheAwareConfig            policies/mod.rs:94-117                        → smgx::CacheAwareConfig
//   struct SelectWorkerInfo            policies/mod.rs:161-175                       → smgx::SelectWorkerInfo
//   trait Worker (the scalars read)    worker/worker.rs:114,151-153,187,208,217      → smgx::Worker / smgx::BasicWorker
//   struct CacheAwarePolicy            policies/cache_aware.rs:74-352, 648-710       → smgx::CacheAwarePolicy
//   kv_index::PositionalIndexer        crates/kv_index/src/event_tree.rs:257-444     → smgx::PositionalIndexer
//   worker::KvEventMonitor (the slice the policy reads + apply_event)                 → smgx::KvEventMonitor
//   struct PrefixHashPolicy / HashRing  policies/prefix_hash.rs:87-235, worker/hash_ring.rs:29-150 → smgx::PrefixHashPolicy / smgx::HashRing
//   struct ConsistentHashingPolicy      policies/consistent_hashing.rs:53-196       → smgx::ConsistentHashingPolicy
// Header-only; link with -lsmgx.  All work happens in the library's CUDA kernels — there is no CPU fallback behind these classes.
#pragma once
#include <cctype>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "smgx.h"

namespace smgx {

struct Error : std::runtime_error {   // SglErrorCode-style status + message (bindings/golang/src/error.rs:6-15)
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
// kv_index::ApplyError (event_tree.rs:88-106)
struct ApplyError : Error { using Error::Error; };

namespace detail {
inline void check(smgx_status st, char* err) {
    std::string msg = err ? err : "";
    if (err) smgx_free_string(err);
    if (st == SMGX_SUCCESS) return;
    if (st == SMGX_WORKER_NOT_TRACKED || st == SMGX_PARENT_BLOCK_NOT_FOUND) throw ApplyError((int)st, msg);
    throw Error((int)st, msg);
}
struct Handle {   // owns one smgx_policy*
    smgx_policy* p = nullptr;
    explicit Handle(const smgx_cache_aware_config& c) {
        char* err = nullptr;
        p = smgx_policy_create(&c, &err);
        if (!p) { std::string m = err ? err : "smgx_policy_create failed"; if (err) smgx_free_string(err); throw Error(SMGX_DEVICE_ERROR, m); }
    }
    ~Handle() { if (p) smgx_policy_free(p); }
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;
};
}  // namespace detail

inline const char* UNKNOWN_MODEL_ID = "unknown";                                                    // crates/protocols/src/lib.rs:8
inline std::string normalize_model_key(const std::string& m) { return m.empty() ? UNKNOWN_MODEL_ID : m; }   // policies/mod.rs:151-157

struct CacheAwareConfig {   // policies/mod.rs:94-117 (+Default)
    float cache_threshold = 0.5f;
    size_t balance_abs_threshold = 32;
    float balance_rel_threshold = 1.1f;
    uint64_t eviction_interval_secs = 30;
    size_t max_tree_size = 10000;
    size_t block_size = 16;
};

class HashRing;
// HeaderMap as (name, value) pairs in insertion order; names compare case-insensitively and get() returns the first value of a name
using HeaderMap = std::vector<std::pair<std::string, std::string>>;

struct SelectWorkerInfo {   // policies/mod.rs:161-175 (headers are read by consistent_hashing only; hash_ring by prefix_hash and consistent_hashing)
    std::optional<std::string> request_text;
    std::optional<std::vector<uint32_t>> tokens;
    std::shared_ptr<HashRing> hash_ring;
    std::optional<HeaderMap> headers;
};

class Worker {   // the scalars CacheAwarePolicy reads through `trait Worker`
public:
    virtual ~Worker() = default;
    virtual const std::string& url() const = 0;
    virtual const std::string& model_id() const = 0;
    virtual size_t load() const = 0;
    virtual bool is_healthy() const = 0;
    virtual bool circuit_breaker_can_execute() const = 0;
    virtual void increment_processed() = 0;
};
class BasicWorker : public Worker {
public:
    explicit BasicWorker(std::string url, std::string model_id = "") : url_(std::move(url)), model_(std::move(model_id)) {}
    const std::string& url() const override { return url_; }
    const std::string& model_id() const override { return model_; }
    size_t load() const override { return load_; }
    bool is_healthy() const override { return healthy_; }
    bool circuit_breaker_can_execute() const override { return circuit_ok_; }
    void increment_processed() override { ++processed_; }
    size_t processed() const { return processed_; }
    void set_load(size_t v) { load_ = v; }
    void set_healthy(bool v) { healthy_ = v; }
    void set_circuit_ok(bool v) { circuit_ok_ = v; }
private:
    std::string url_, model_;
    size_t load_ = 0, processed_ = 0;
    bool healthy_ = true, circuit_ok_ = true;
};
using Workers = std::vector<std::shared_ptr<Worker>>;

struct StoredBlock { uint64_t seq_hash, content_hash; };   // event_tree.rs:81-86
struct OverlapScores { std::map<uint32_t, uint32_t> scores; std::map<uint32_t, uint64_t> tree_sizes; };   // :112-118

class PositionalIndexer {   // bound to (policy handle, model); the caller-owned WorkerBlockMap lives inside the library per worker id
public:
    PositionalIndexer(std::shared_ptr<detail::Handle> h, std::string model, uint32_t jump_size) : h_(std::move(h)), model_(std::move(model)) {
        if (jump_size == 0) throw std::invalid_argument("jump_size must be greater than 0");   // event_tree.rs:280
        call(smgx_indexer_create, jump_size);
    }
    uint32_t intern_worker(const std::string& url) { uint32_t id = 0; call(smgx_indexer_intern_worker, url.c_str(), &id); return id; }   // :509-525
    std::optional<uint32_t> worker_id(const std::string& url) {                                                                          // :294
        int64_t id = -1; call(smgx_indexer_worker_id, url.c_str(), &id);
        return id < 0 ? std::nullopt : std::optional<uint32_t>((uint32_t)id);
    }
    void apply_stored(uint32_t worker, const std::vector<StoredBlock>& blocks, std::optional<uint64_t> parent = std::nullopt) {          // :305-366
        std::vector<uint64_t> seq(blocks.size()), con(blocks.size());
        for (size_t i = 0; i < blocks.size(); ++i) { seq[i] = blocks[i].seq_hash; con[i] = blocks[i].content_hash; }
        const uint64_t par = parent.value_or(0);
        call(smgx_indexer_apply_stored, worker, seq.data(), con.data(), (uint32_t)blocks.size(), parent ? &par : nullptr);
    }
    // same, hashing the blocks' token ids on the GPU like convert_kv_block (kv_event_monitor.rs:592-597)
    void apply_stored_tokens(uint32_t worker, const std::vector<uint64_t>& seq_hashes, const std::vector<uint32_t>& token_ids, uint32_t block_size,
                             std::optional<uint64_t> parent = std::nullopt) {
        if (token_ids.size() != seq_hashes.size() * (size_t)block_size) throw std::invalid_argument("token_ids must hold block_size ids per block");
        const uint64_t par = parent.value_or(0);
        call(smgx_indexer_apply_stored_tokens, worker, seq_hashes.data(), token_ids.data(), block_size, (uint32_t)seq_hashes.size(), parent ? &par : nullptr);
    }
    void apply_removed(uint32_t worker, const std::vector<uint64_t>& seq_hashes) { call(smgx_indexer_apply_removed, worker, seq_hashes.data(), (uint32_t)seq_hashes.size()); }
    void apply_cleared(uint32_t worker) { call(smgx_indexer_apply_cleared, worker); }
    void remove_worker(uint32_t worker) { call(smgx_indexer_remove_worker, worker); }
    size_t current_size() { uint64_t v = 0; call(smgx_indexer_current_size, &v); return (size_t)v; }
    OverlapScores find_matches(const std::vector<uint64_t>& content_hashes, bool early_exit = false) {                                     // :461 (GPU kernel)
        std::vector<uint32_t> sc(2048); std::vector<uint64_t> ts(2048); uint32_t nw = 0;
        call(smgx_indexer_find_matches, content_hashes.data(), (uint32_t)content_hashes.size(), early_exit ? 1 : 0, sc.data(), ts.data(), 2048u, &nw);
        OverlapScores o;
        for (uint32_t i = 0; i < nw; ++i) if (sc[i]) { o.scores[i] = sc[i]; o.tree_sizes[i] = ts[i]; }
        return o;
    }
    const std::string& model() const { return model_; }
private:
    template <class F, class... A> void call(F f, A... a) { char* err = nullptr; detail::check(f(h_->p, model_.c_str(), a..., &err), err); }
    std::shared_ptr<detail::Handle> h_;
    std::string model_;
};

// proto KvCacheEvent (crates/grpc_client/proto/common.proto:41-58), flattened
struct KvBlock { int64_t block_hash; std::vector<uint32_t> token_ids; uint32_t block_size = 0; };
struct KvCacheEvent {
    enum Kind { Stored, Removed, Cleared } kind = Stored;
    std::vector<KvBlock> blocks;                  // Stored
    std::optional<int64_t> parent_block_hash;     // Stored
    std::vector<int64_t> block_hashes;            // Removed
};

class KvEventMonitor {   // per-model indexers, learned block sizes, apply_event (worker/kv_event_monitor.rs)
public:
    explicit KvEventMonitor(std::shared_ptr<detail::Handle> h) : h_(std::move(h)) {}
    std::shared_ptr<PositionalIndexer> create_indexer(const std::string& model, uint32_t jump_size = 64) {   // DEFAULT_JUMP_SIZE :31
        auto ix = std::make_shared<PositionalIndexer>(h_, model, jump_size);
        indexers_[model] = ix;
        return ix;
    }
    std::shared_ptr<PositionalIndexer> get_indexer(const std::string& model) const { auto it = indexers_.find(model); return it == indexers_.end() ? nullptr : it->second; }
    void set_block_size(const std::string& model, uint32_t bs) { char* err = nullptr; detail::check(smgx_indexer_set_block_size(h_->p, model.c_str(), bs, &err), err); }
    // one KvEventBatch of a worker's stream (process_stream :513-517 → apply_event :525-597); returns the fresh-chain fallbacks
    uint32_t apply_events(const std::string& model, uint32_t worker_id, const std::vector<KvCacheEvent>& events) {
        std::vector<smgx_kv_event> evs;
        std::vector<int64_t> hashes;
        std::vector<uint32_t> toks, offs{0};
        for (const auto& ev : events) {
            smgx_kv_event e{};
            e.worker_id = worker_id;
            e.first_block = (uint32_t)hashes.size();
            if (ev.kind == KvCacheEvent::Stored) {
                e.kind = SMGX_KV_STORED; e.n_blocks = (uint32_t)ev.blocks.size();
                e.has_parent = ev.parent_block_hash ? 1 : 0; e.parent_block_hash = ev.parent_block_hash.value_or(0);
                if (!ev.blocks.empty() && !learned_[model] && ev.blocks[0].block_size > 0) { set_block_size(model, ev.blocks[0].block_size); learned_[model] = true; }   // :270-296
                for (const auto& b : ev.blocks) { hashes.push_back(b.block_hash); toks.insert(toks.end(), b.token_ids.begin(), b.token_ids.end()); offs.push_back((uint32_t)toks.size()); }
            } else if (ev.kind == KvCacheEvent::Removed) {
                e.kind = SMGX_KV_REMOVED; e.n_blocks = (uint32_t)ev.block_hashes.size();
                for (int64_t hsh : ev.block_hashes) { hashes.push_back(hsh); offs.push_back((uint32_t)toks.size()); }
            } else e.kind = SMGX_KV_CLEARED;
            evs.push_back(e);
        }
        uint32_t fallbacks = 0;
        char* err = nullptr;
        detail::check(smgx_kv_events_apply(h_->p, model.c_str(), evs.data(), (uint32_t)evs.size(), hashes.data(), offs.data(), toks.data(), (uint32_t)hashes.size(),
                                           &fallbacks, &err), err);
        return fallbacks;
    }
private:
    std::shared_ptr<detail::Handle> h_;
    std::map<std::string, std::shared_ptr<PositionalIndexer>> indexers_;
    std::map<std::string, bool> learned_;
};

class LoadBalancingPolicy {   // policies/mod.rs:43-86
public:
    virtual ~LoadBalancingPolicy() = default;
    virtual std::optional<size_t> select_worker(const Workers& workers, const SelectWorkerInfo& info) = 0;   // index into the GIVEN slice; nullopt = None
    virtual void on_request_complete(const std::string& worker_url, bool success) {}
    virtual const char* name() const = 0;
    virtual bool needs_request_text() const { return false; }
};

struct Decision { int32_t idx; smgx_decision_info info; };
class StringTree;

class CacheAwarePolicy : public LoadBalancingPolicy {   // policies/cache_aware.rs:74-352, 648-710
public:
    explicit CacheAwarePolicy(const CacheAwareConfig& config = CacheAwareConfig(), int device_id = 0, uint32_t max_batch = 0, uint32_t max_tokens_per_request = 0,
                              smgx_tree_batch_mode mode = SMGX_TREE_BATCH_SEQUENTIAL)
        : config_(config) {
        smgx_cache_aware_config c;
        smgx_default_config(&c);
        c.cache_threshold = config.cache_threshold; c.balance_abs_threshold = config.balance_abs_threshold; c.balance_rel_threshold = config.balance_rel_threshold;
        c.eviction_interval_secs = config.eviction_interval_secs; c.max_tree_size = config.max_tree_size; c.block_size = config.block_size;
        c.device_id = device_id; c.max_batch = max_batch; c.max_tokens_per_request = max_tokens_per_request; c.tree_batch_mode = mode;
        h_ = std::make_shared<detail::Handle>(c);
    }
    static CacheAwarePolicy with_config(const CacheAwareConfig& c) { return CacheAwarePolicy(c); }   // cache_aware.rs:120

    const char* name() const override { return smgx_policy_name(); }     // "cache_aware" (:704-706)
    bool needs_request_text() const override { return true; }            // :708-710
    void on_request_complete(const std::string&, bool) override {}       // :692-702 (no state)

    void init_workers(const Workers& workers) {                          // :219-249
        std::map<std::string, std::vector<std::string>> by_model;
        for (auto& w : workers) by_model[normalize_model_key(w->model_id())].push_back(w->url());
        for (auto& kv : by_model) register_slice(kv.first, kv.second);
    }
    void add_worker(const Worker& w) { char* err = nullptr; detail::check(smgx_add_worker(h_->p, normalize_model_key(w.model_id()).c_str(), w.url().c_str(), &err), err); }   // :252-266
    void remove_worker_by_url(const std::string& url) { char* err = nullptr; detail::check(smgx_remove_worker(h_->p, "", url.c_str(), &err), err); }                            // :302-308 (no-op)
    void evict_cache(size_t max_size) { char* err = nullptr; detail::check(smgx_evict_cache(h_->p, max_size, &err), err); }                                                      // :311-352
    // Batches as the request stream of a router that guards every cache_aware pick (WorkerLoadGuard): request i sees the fleet snapshot
    // plus the picks of requests < i, in every mode (event-driven, token tree, string tree).  Needs SMGX_TREE_BATCH_SEQUENTIAL.
    void set_load_feedback_all_modes(bool enabled) {
        char* err = nullptr; detail::check(smgx_set_load_feedback_policies(h_->p, enabled ? SMGX_FEEDBACK_CACHE_AWARE : 0u, &err), err);
    }

    std::shared_ptr<KvEventMonitor> kv_event_monitor() { return std::make_shared<KvEventMonitor>(h_); }
    void set_kv_event_monitor(std::shared_ptr<KvEventMonitor> m) {       // :213-215
        monitor_ = std::move(m);
        char* err = nullptr; detail::check(smgx_set_kv_event_monitor(h_->p, monitor_ ? 1 : 0, &err), err);
    }

    // LoadBalancingPolicy::select_worker (:648-690): index into `workers` or nullopt
    std::optional<size_t> select_worker(const Workers& workers, const SelectWorkerInfo& info) override {
        if (workers.empty()) return std::nullopt;
        Decision d;
        if (info.tokens) d = select_worker_batch(workers, {*info.tokens})[0];
        else d = select_worker_batch_request_text(workers, {info.request_text.value_or("")})[0];   // :688-689
        if (d.idx < 0) return std::nullopt;
        workers[(size_t)d.idx]->increment_processed();   // mirror of increment_processed(); the library keeps the authoritative counters
        return (size_t)d.idx;
    }
    // batched forms: every request sees one fleet snapshot
    std::vector<Decision> select_worker_batch(const Workers& workers, const std::vector<std::vector<uint32_t>>& requests) {
        const std::string model = push_fleet(workers);
        std::vector<uint32_t> toks, offs{0};
        for (auto& r : requests) { toks.insert(toks.end(), r.begin(), r.end()); offs.push_back((uint32_t)toks.size()); }
        if (toks.empty()) toks.push_back(0);
        std::vector<int32_t> idx(requests.size(), -1);
        std::vector<smgx_decision_info> info(requests.size());
        char* err = nullptr;
        detail::check(smgx_select_batch_tokens(h_->p, model.c_str(), toks.data(), offs.data(), (uint32_t)requests.size(), idx.data(), info.data(), &err), err);
        return zip(idx, info);
    }
    std::vector<Decision> select_worker_batch_request_text(const Workers& workers, const std::vector<std::string>& texts) {
        const std::string model = push_fleet(workers);
        std::string blob;
        std::vector<uint32_t> offs{0};
        for (auto& t : texts) { blob += t; offs.push_back((uint32_t)blob.size()); }
        if (blob.empty()) blob.push_back('\0');
        std::vector<int32_t> idx(texts.size(), -1);
        std::vector<smgx_decision_info> info(texts.size());
        char* err = nullptr;
        detail::check(smgx_select_batch_request_text(h_->p, model.c_str(), (const uint8_t*)blob.data(), offs.data(), (uint32_t)texts.size(), idx.data(), info.data(), &err), err);
        return zip(idx, info);
    }
    std::shared_ptr<detail::Handle> handle() const { return h_; }
    std::shared_ptr<StringTree> string_tree(const std::string& model = UNKNOWN_MODEL_ID);   // string_trees[model] (cache_aware.rs:78)

private:
    static std::vector<Decision> zip(const std::vector<int32_t>& idx, const std::vector<smgx_decision_info>& info) {
        std::vector<Decision> out(idx.size());
        for (size_t i = 0; i < idx.size(); ++i) out[i] = Decision{idx[i], info[i]};
        return out;
    }
    void register_slice(const std::string& model, const std::vector<std::string>& urls) {
        std::vector<const char*> c;
        for (auto& u : urls) c.push_back(u.c_str());
        char* err = nullptr;
        detail::check(smgx_set_workers(h_->p, model.c_str(), c.data(), (uint32_t)c.size(), &err), err);
        slices_[model] = urls;
    }
    // model of the first healthy worker (:659), the URL slice when it changed, and the per-request scalars (worker.rs:151-153,187,208)
    std::string push_fleet(const Workers& workers) {
        std::string model = workers.empty() ? UNKNOWN_MODEL_ID : normalize_model_key(workers[0]->model_id());
        for (auto& w : workers) if (w->is_healthy() && w->circuit_breaker_can_execute()) { model = normalize_model_key(w->model_id()); break; }
        std::vector<std::string> urls;
        for (auto& w : workers) urls.push_back(w->url());
        auto it = slices_.find(model);
        if (it == slices_.end() || it->second != urls) register_slice(model, urls);
        std::vector<uint64_t> loads;
        std::vector<uint8_t> healthy, circuit;
        for (auto& w : workers) { loads.push_back(w->load()); healthy.push_back(w->is_healthy()); circuit.push_back(w->circuit_breaker_can_execute()); }
        char* err = nullptr;
        detail::check(smgx_set_fleet_state(h_->p, model.c_str(), loads.data(), healthy.data(), circuit.data(), (uint32_t)workers.size(), &err), err);
        return model;
    }
    CacheAwareConfig config_;
    std::shared_ptr<detail::Handle> h_;
    std::shared_ptr<KvEventMonitor> monitor_;
    std::map<std::string, std::vector<std::string>> slices_;
};

// kv_index::Tree (char-level string tree, HTTP text routing) of one model: writers on the host-authoritative tree inside the library,
// including the mesh wire format (crates/kv_index/src/snapshot.rs; string_tree.rs:1052-1578)
class StringTree {
public:
    StringTree(std::shared_ptr<detail::Handle> h, std::string model = UNKNOWN_MODEL_ID) : h_(std::move(h)), model_(std::move(model)) {}
    void insert_text(const std::string& text, const std::string& tenant) {                  // :393-557
        call(smgx_stree_insert_text, (const uint8_t*)text.data(), (uint32_t)text.size(), tenant.c_str());
    }
    size_t node_count() { uint64_t n = 0; call(smgx_stree_node_count, &n); return (size_t)n; }
    void clear() { call(smgx_stree_clear); }
    std::string snapshot_bytes() {                                                            // Tree::snapshot().to_bytes()
        char* out = nullptr; uint64_t len = 0;
        call(smgx_stree_snapshot, &out, &len);
        std::string b(out, (size_t)len);
        smgx_free_string(out);
        return b;
    }
    void load_snapshot(const std::string& bytes) { call(smgx_stree_load_snapshot, (const uint8_t*)bytes.data(), (uint64_t)bytes.size()); }    // Tree::from_snapshot
    void merge_snapshot(const std::string& bytes) { call(smgx_stree_merge_snapshot, (const uint8_t*)bytes.data(), (uint64_t)bytes.size()); }  // Tree::merge_snapshot
private:
    template <class F, class... A> void call(F f, A... a) { char* err = nullptr; detail::check(f(h_->p, model_.c_str(), a..., &err), err); }
    std::shared_ptr<detail::Handle> h_;
    std::string model_;
};

inline std::shared_ptr<StringTree> CacheAwarePolicy::string_tree(const std::string& model) { return std::make_shared<StringTree>(h_, normalize_model_key(model)); }

// ---- adjacent policy on the same plumbing: prefix_hash (policies/prefix_hash.rs) over worker::HashRing (worker/hash_ring.rs) ----
struct PrefixHashConfig {   // prefix_hash.rs:38-58
    size_t prefix_token_count = 256;
    double load_factor = 1.25;
};

class HashRing {   // per-model ring, built (hashed + sorted) inside the library
public:
    HashRing(std::shared_ptr<detail::Handle> h, std::string model, const std::vector<std::string>& urls) : h_(std::move(h)), model_(std::move(model)), urls_(urls) {
        std::vector<const char*> c;
        for (auto& u : urls_) c.push_back(u.c_str());
        char* err = nullptr;
        detail::check(smgx_hash_ring_set(h_->p, model_.c_str(), c.data(), (uint32_t)c.size(), &err), err);
    }
    size_t len() const { uint32_t n = 0; char* err = nullptr; detail::check(smgx_hash_ring_entries(h_->p, model_.c_str(), nullptr, nullptr, 0, &n, &err), err); return n; }   // :142-144
    bool is_empty() const { return len() == 0; }
    size_t worker_count() const { return len() / 150; }   // :147-149
    // find_healthy_url (:102-134); the predicate is evaluated once per ring URL, the walk runs on the GPU
    template <class F> std::optional<std::string> find_healthy_url(const std::string& key, F is_healthy) const {
        std::vector<uint8_t> ok(urls_.size() ? urls_.size() : 1, 0);
        for (size_t u = 0; u < urls_.size(); ++u) ok[u] = is_healthy(urls_[u]) ? 1 : 0;
        const uint32_t offs[2] = {0, (uint32_t)key.size()};
        int32_t out = -1;
        char* err = nullptr;
        detail::check(smgx_hash_ring_find_healthy(h_->p, model_.c_str(), (const uint8_t*)key.data(), offs, 1, ok.data(), &out, &err), err);
        return out < 0 ? std::nullopt : std::optional<std::string>(urls_[(size_t)out]);
    }
    const std::string& model() const { return model_; }
    const std::shared_ptr<detail::Handle>& handle() const { return h_; }
private:
    std::shared_ptr<detail::Handle> h_;
    std::string model_;
    std::vector<std::string> urls_;
};

class PrefixHashPolicy : public LoadBalancingPolicy {   // prefix_hash.rs:87-235
public:
    explicit PrefixHashPolicy(const PrefixHashConfig& config = PrefixHashConfig(), int device_id = 0, uint32_t max_batch = 0) : config_(config) {
        smgx_cache_aware_config c;
        smgx_default_config(&c);
        c.eviction_interval_secs = 0; c.device_id = device_id; c.max_batch = max_batch;
        h_ = std::make_shared<detail::Handle>(c);
        char* err = nullptr;
        detail::check(smgx_prefix_hash_configure(h_->p, config.prefix_token_count, config.load_factor, &err), err);
    }
    static PrefixHashPolicy with_defaults() { return PrefixHashPolicy(); }   // :100-103
    // batches as the request stream of a router that guards every pick (gRPC): the bound and the fallback read the running loads
    void set_load_feedback(bool enabled) {
        char* err = nullptr; detail::check(smgx_set_load_feedback_policies(h_->p, enabled ? SMGX_FEEDBACK_PREFIX_HASH : 0u, &err), err);
    }
    const char* name() const override { return "prefix_hash"; }              // :231-233
    // the registry's per-model ring (SelectWorkerInfo.hash_ring), bound to this policy's device state
    std::shared_ptr<HashRing> hash_ring(const std::vector<std::string>& urls, const std::string& model = UNKNOWN_MODEL_ID) {
        return std::make_shared<HashRing>(h_, normalize_model_key(model), urls);
    }
    std::vector<Decision> select_worker_batch(const Workers& workers, const std::vector<std::optional<std::vector<uint32_t>>>& requests,
                                              const std::shared_ptr<HashRing>& ring) {
        if (ring && ring->handle() != h_) throw std::invalid_argument("hash ring belongs to another policy: build it with PrefixHashPolicy::hash_ring()");
        const std::string model = ring ? ring->model() : normalize_model_key(workers.empty() ? "" : workers[0]->model_id());
        char* err = nullptr;
        if (!ring) detail::check(smgx_hash_ring_clear(h_->p, model.c_str(), &err), err);
        std::vector<std::string> urls;
        for (auto& w : workers) urls.push_back(w->url());
        auto it = slices_.find(model);
        if (it == slices_.end() || it->second != urls) {
            std::vector<const char*> c;
            for (auto& u : urls) c.push_back(u.c_str());
            detail::check(smgx_set_workers(h_->p, model.c_str(), c.data(), (uint32_t)c.size(), &err), err);
            slices_[model] = urls;
        }
        std::vector<uint64_t> loads;
        std::vector<uint8_t> healthy;
        for (auto& w : workers) { loads.push_back(w->load()); healthy.push_back(w->is_healthy()); }   // only load() and is_healthy() are read (:140, :148)
        detail::check(smgx_set_fleet_state(h_->p, model.c_str(), loads.data(), healthy.data(), nullptr, (uint32_t)workers.size(), &err), err);
        std::vector<uint32_t> toks, offs{0};
        std::vector<uint8_t> has;
        for (auto& r : requests) { if (r) toks.insert(toks.end(), r->begin(), r->end()); has.push_back(r ? 1 : 0); offs.push_back((uint32_t)toks.size()); }
        if (toks.empty()) toks.push_back(0);
        std::vector<int32_t> idx(requests.size(), -1);
        std::vector<smgx_decision_info> info(requests.size());
        detail::check(smgx_prefix_hash_select_batch_tokens(h_->p, model.c_str(), toks.data(), offs.data(), (uint32_t)requests.size(), has.data(), idx.data(), info.data(),
                                                           &err), err);
        std::vector<Decision> out(idx.size());
        for (size_t i = 0; i < idx.size(); ++i) out[i] = Decision{idx[i], info[i]};
        return out;
    }
    // LoadBalancingPolicy::select_worker (:225-229)
    std::optional<size_t> select_worker(const Workers& workers, const SelectWorkerInfo& info) override {
        const Decision d = select_worker_batch(workers, {info.tokens}, info.hash_ring)[0];
        return d.idx < 0 ? std::nullopt : std::optional<size_t>((size_t)d.idx);
    }
private:
    PrefixHashConfig config_;
    std::shared_ptr<detail::Handle> h_;
    std::map<std::string, std::vector<std::string>> slices_;
};

class PowerOfTwoPolicy : public LoadBalancingPolicy {   // power_of_two.rs:18-135
public:
    explicit PowerOfTwoPolicy(int device_id = 0, uint32_t max_batch = 0, uint64_t seed = 0x5EED) : seed_(seed) {
        smgx_cache_aware_config c;
        smgx_default_config(&c);
        c.eviction_interval_secs = 0; c.device_id = device_id; c.max_batch = max_batch;
        h_ = std::make_shared<detail::Handle>(c);
    }
    const char* name() const override { return "power_of_two"; }             // :122-124
    // batches as the request stream of a router that guards every pick (gRPC): the request-count comparison reads the running loads
    void set_load_feedback(bool enabled) {
        char* err = nullptr; detail::check(smgx_set_load_feedback_policies(h_->p, enabled ? SMGX_FEEDBACK_POWER_OF_TWO : 0u, &err), err);
    }
    // update_loads (:129-135): url → WorkerLoadResponse::effective_token_usage() (the mean token_usage over the DP ranks; 0.0 for none)
    void update_loads(const std::map<std::string, double>& token_usage) {
        if (token_usage.empty()) return;
        std::vector<const char*> urls;
        std::vector<double> v;
        for (auto& kv : token_usage) { urls.push_back(kv.first.c_str()); v.push_back(kv.second); }
        char* err = nullptr;
        detail::check(smgx_power_of_two_update_loads(h_->p, urls.data(), v.data(), (uint32_t)urls.size(), &err), err);
    }
    // n requests against one snapshot of the slice; every call consumes one value of the policy's seed sequence
    std::vector<int32_t> select_worker_batch(const Workers& workers, uint32_t n) {
        const std::string model = normalize_model_key(workers.empty() ? "" : workers[0]->model_id());
        char* err = nullptr;
        std::vector<std::string> urls;
        for (auto& w : workers) urls.push_back(w->url());
        auto it = slices_.find(model);
        if (it == slices_.end() || it->second != urls) {
            std::vector<const char*> c;
            for (auto& u : urls) c.push_back(u.c_str());
            detail::check(smgx_set_workers(h_->p, model.c_str(), c.data(), (uint32_t)c.size(), &err), err);
            slices_[model] = urls;
        }
        std::vector<uint64_t> loads;
        std::vector<uint8_t> healthy, circuit;
        for (auto& w : workers) { loads.push_back(w->load()); healthy.push_back(w->is_healthy()); circuit.push_back(w->circuit_breaker_can_execute()); }
        detail::check(smgx_set_fleet_state(h_->p, model.c_str(), loads.data(), healthy.data(), circuit.data(), (uint32_t)workers.size(), &err), err);
        std::vector<int32_t> idx(n, -1);
        std::vector<int32_t> pairs(2 * (size_t)n, -1);
        ++calls_;
        detail::check(smgx_power_of_two_select_batch(h_->p, model.c_str(), n, seed_ + 0xD1B54A32D192ED03ULL * calls_, idx.data(), pairs.data(), nullptr, &err), err);
        for (uint32_t i = 0; i < n; ++i) if (idx[i] >= 0 && pairs[2 * (size_t)i] >= 0) workers[(size_t)idx[i]]->increment_processed();   // :110 (not on the single-worker return)
        return idx;
    }
    std::optional<size_t> select_worker(const Workers& workers, const SelectWorkerInfo&) override {   // :36-120
        if (workers.empty()) return std::nullopt;
        const int32_t i = select_worker_batch(workers, 1)[0];
        return i < 0 ? std::nullopt : std::optional<size_t>((size_t)i);
    }
private:
    std::shared_ptr<detail::Handle> h_;
    std::map<std::string, std::vector<std::string>> slices_;
    uint64_t seed_, calls_ = 0;
};

class ConsistentHashingPolicy : public LoadBalancingPolicy {   // consistent_hashing.rs:53-196
public:
    explicit ConsistentHashingPolicy(int device_id = 0, uint32_t max_batch = 0, uint64_t seed = 0x5EED) : seed_(seed) {
        smgx_cache_aware_config c;
        smgx_default_config(&c);
        c.eviction_interval_secs = 0; c.device_id = device_id; c.max_batch = max_batch;
        h_ = std::make_shared<detail::Handle>(c);
    }
    const char* name() const override { return "consistent_hashing"; }      // :188-190
    // the registry's per-model ring, bound to this policy's device state
    std::shared_ptr<HashRing> hash_ring(const std::vector<std::string>& urls, const std::string& model = "unknown") {
        return std::make_shared<HashRing>(h_, normalize_model_key(model), urls);
    }
    struct Batch { std::vector<int32_t> idx; std::vector<uint8_t> branch; std::vector<uint64_t> key_pos; };   // branch: smgx_ch_branch
    // one batch against one snapshot of the slice (headers[i] = std::nullopt: info.headers = None); every call consumes one value of the
    // policy's seed sequence, request i uses draw i of it
    Batch select_worker_batch(const Workers& workers, const std::vector<std::optional<HeaderMap>>& headers, const std::shared_ptr<HashRing>& ring = nullptr) {
        static const char* const kNames[5] = {"x-smg-target-worker", "x-smg-routing-key", "authorization", "x-forwarded-for", "cookie"};
        std::string model = ring ? ring->model() : normalize_model_key(workers.empty() ? "" : workers[0]->model_id());
        if (ring && ring->handle() != h_) throw Error(SMGX_INVALID_ARGUMENT, "hash ring belongs to another policy: build it with ConsistentHashingPolicy::hash_ring()");
        char* err = nullptr;
        if (!ring && ringed_.count(model)) { detail::check(smgx_hash_ring_clear(h_->p, model.c_str(), &err), err); ringed_.erase(model); }
        if (ring) ringed_.insert(model);
        std::vector<std::string> urls;
        for (auto& w : workers) urls.push_back(w->url());
        auto it = slices_.find(model);
        if (it == slices_.end() || it->second != urls) {
            std::vector<const char*> c;
            for (auto& u : urls) c.push_back(u.c_str());
            detail::check(smgx_set_workers(h_->p, model.c_str(), c.data(), (uint32_t)c.size(), &err), err);
            slices_[model] = urls;
        }
        std::vector<uint64_t> loads;
        std::vector<uint8_t> healthy, circuit;
        for (auto& w : workers) { loads.push_back(w->load()); healthy.push_back(w->is_healthy()); circuit.push_back(w->circuit_breaker_can_execute()); }
        detail::check(smgx_set_fleet_state(h_->p, model.c_str(), loads.data(), healthy.data(), circuit.data(), (uint32_t)workers.size(), &err), err);
        const uint32_t n = (uint32_t)headers.size();
        std::string values;
        std::vector<uint32_t> offsets{0};
        std::vector<uint8_t> present(n, 0);
        for (uint32_t i = 0; i < n; ++i)
            for (int h = 0; h < 5; ++h) {
                if (headers[i])
                    for (auto& kv : *headers[i]) {
                        if (!iequals(kv.first, kNames[h])) continue;
                        present[i] |= (uint8_t)(1u << h); values += kv.second;
                        break;
                    }
                offsets.push_back((uint32_t)values.size());
            }
        Batch b{std::vector<int32_t>(n, -1), std::vector<uint8_t>(n, 0), std::vector<uint64_t>(n, 0)};
        ++calls_;
        detail::check(smgx_consistent_hashing_select_batch(h_->p, model.c_str(), n, (const uint8_t*)values.data(), offsets.data(), present.data(),
                                                           seed_ + 0xD1B54A32D192ED03ULL * calls_, b.idx.data(), b.branch.data(), b.key_pos.data(), &err), err);
        return b;
    }
    std::pair<std::optional<size_t>, smgx_ch_branch> select_worker_impl(const Workers& workers, const SelectWorkerInfo& info) {   // :116-180
        const Batch b = select_worker_batch(workers, {info.headers}, info.hash_ring);
        return {b.idx[0] < 0 ? std::nullopt : std::optional<size_t>((size_t)b.idx[0]), (smgx_ch_branch)b.branch[0]};
    }
    std::optional<size_t> select_worker(const Workers& workers, const SelectWorkerInfo& info) override { return select_worker_impl(workers, info).first; }   // :182-186
private:
    static bool iequals(const std::string& a, const char* b) {
        size_t i = 0;
        for (; i < a.size() && b[i]; ++i) if (std::tolower((unsigned char)a[i]) != b[i]) return false;
        return i == a.size() && !b[i];
    }
    std::shared_ptr<detail::Handle> h_;
    std::map<std::string, std::vector<std::string>> slices_;
    std::set<std::string> ringed_;
    uint64_t seed_, calls_ = 0;
};

}  // namespace smgx
