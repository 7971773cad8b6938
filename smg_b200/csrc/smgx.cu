// smgx policy object + C ABI (include/smgx.h).
//
// Host-side counterpart of CacheAwarePolicy (model_gateway/src/policies/cache_aware.rs:74-101): per-model state
// keyed by normalize_model_key (policies/mod.rs:151-157), the fleet snapshot select_worker reads from `dyn Worker`
// (worker/worker.rs:151-153,187,208), the KV-event indexers a KvEventMonitor would own, and a small ring of
// stream "lanes" that stage request batches into HBM and run the kernels.  Every decision is produced by the
// kernels in event_kernels.cu; nothing here computes a pick on the CPU.
#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "common.h"
#include "event_index.h"
#include "kernels.h"
#include "tokenizer.h"
#include "token_tree.h"
#include "string_tree.h"
#include "blake3.h"
#include "prefix_hash.h"
#include "power_of_two.h"
#include "consistent_hashing.h"
#include <cstdio>
#include <cctype>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <unordered_map>
#include <unordered_set>

namespace smgx {

static std::string norm_model(const char* m) { return (m == nullptr || m[0] == 0) ? std::string("unknown") : std::string(m); }

struct ModelState {
    // the `&[Arc<dyn Worker>]` slice, in slice order
    std::vector<std::string> urls;
    std::vector<uint64_t> loads;
    std::vector<uint8_t> flags;      // bit0 is_healthy(), bit1 circuit_breaker_can_execute()
    std::vector<uint64_t> processed; // increment_processed() per slice index
    uint64_t slice_version = 0;      // bumped by smgx_set_workers: a ticket credits `processed` only against the slice it was decided on
    // KvEventMonitor state for this model
    std::unique_ptr<EventIndex> indexer;
    std::unique_ptr<Tokenizer> tokenizer;   // TokenizerRegistry entry for this model
    std::unique_ptr<TokenTreeIndex> token_tree;   // token_trees[model] (cache_aware.rs:79)
    std::unique_ptr<StringTreeIndex> string_tree; // string_trees[model] (cache_aware.rs:78)
    // hash_index[model] (cache_aware.rs:95-101): blake3 path hash of the full request → copy of the matched prefix
    // values live in append-only arenas (one allocation-free copy per routed request); an overwritten entry's old bytes are
    // reclaimed when evict_cache clears the map
    std::unordered_map<uint64_t, std::pair<uint64_t, uint32_t>> hash_index_tokens, hash_index_text;   // hash → (arena offset, length)
    std::vector<uint32_t> hash_arena_tokens;
    std::string hash_arena_text;
    uint64_t hash_dead_tokens = 0, hash_dead_text = 0;   // arena elements / bytes no entry points at any more
    DevBuf d_slice_of_tenant;
    std::vector<int32_t> slice_of_tenant;         // host copy of d_slice_of_tenant (the load-feedback decision of the tree modes)
    std::vector<uint32_t> tenant_of_slice;        // tenant id of urls[i]
    uint64_t seen_tenants_version = ~0ULL;
    bool has_learned_bs = false;
    uint32_t learned_bs = 0;
    // device copy of the fleet
    DevBuf d_loads, d_flags, d_id_of_slice, d_derived, d_slice_of_id, d_load_of_id, d_elig;
    bool fleet_dirty = true;
    bool fleet_has_dups = false;   // two slice entries share a URL
    bool fleet_dirty_tenant = true;
    uint64_t seen_workers_version = ~0ULL;
    // prefix_hash policy (policies/prefix_hash.rs): info.hash_ring of this model (worker/hash_ring.rs) and its device copies
    bool has_ring = false;
    std::vector<std::string> ring_urls;
    std::vector<uint64_t> ring_pos;       // sorted positions
    std::vector<uint32_t> ring_url;       // entry → index into ring_urls
    DevBuf d_ring_pos, d_ring_slice, d_ring_url, d_ring_bucket, d_dup_prev, d_pf_loads, d_pf_flags, d_pf_derived;
    uint32_t ring_bucket_shift = 63;
    bool pf_struct_dirty = true;          // slice or ring changed: entry → slice map must be rebuilt
    bool pf_state_dirty = true;           // loads / health changed: fleet summary must be recomputed
    // consistent_hashing policy (policies/consistent_hashing.rs): per fleet snapshot, the ascending is_healthy() indices followed by the
    // ascending values of the healthy URL → last healthy index map
    DevBuf d_ch_lists;
    std::vector<int32_t> ch_lists;
    uint32_t ch_n_healthy = 0;
    bool ch_dirty = true;
};

struct Lane {
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr, t0 = nullptr, t1 = nullptr;
    DevBuf d_fb;   // load-feedback scratch: per-request tied sets + scores
    DevBuf d_slowq;   // queue between event_lane_kernel / event_warp_kernel and event_slow_kernel
    DevBuf d_recs;    // SearchRec per request: hash kernel → search kernel
    DevBuf d_groups;  // event_hs_kernel's arrival counters, [kMaxMultiBatches][group_stride] (zeroed once; self-resetting)
    uint32_t group_stride = 0;
    // concurrent split launch (hash on `stream`, search on `side`): device counters the hash CTAs count into + their host-side running totals
    cudaStream_t side = nullptr;
    cudaEvent_t pre = nullptr, side_done = nullptr;
    DevBuf d_ready;
    uint32_t ready_cum[kMaxMultiBatches] = {};
    DevBuf d_tokens, d_offsets, d_out, d_info, d_hash, d_text, d_toff, d_path, d_path_len, d_tenant, d_path_tenant, d_fill, d_chunk_start, d_cv, d_hashes;
    Tokenizer::Scratch tok_scratch;
    bool busy = false;
    bool has_done = false;
    uint64_t ticket = 0;
    // completion bookkeeping for the host-buffer API
    ModelState* model = nullptr;
    const int32_t* host_out = nullptr;
    uint32_t n = 0;
    uint64_t slice_version = 0;   // ModelState::slice_version at submission
    // load-feedback bookkeeping of a host-buffer submission (see Policy::wait)
    const uint32_t* fb_tokens = nullptr;
    const uint32_t* fb_offsets = nullptr;
    smgx_decision_info* fb_info_host = nullptr;
    std::vector<smgx_decision_info> fb_info;
};

class Policy {
public:
    explicit Policy(const smgx_cache_aware_config& c) : cfg(c) {
        if (cfg.max_batch == 0) cfg.max_batch = 65536;
        if (cfg.max_tokens_per_request == 0) cfg.max_tokens_per_request = 32768;
        tree_batch_mode = cfg.tree_batch_mode == SMGX_TREE_BATCH_SNAPSHOT ? SMGX_TREE_BATCH_SNAPSHOT : SMGX_TREE_BATCH_SEQUENTIAL;
        if (cfg.device_id >= 0) {
            int count = 0;
            cudaError_t e = cudaGetDeviceCount(&count);
            if (e != cudaSuccess || count == 0)
                throw Error(SMGX_DEVICE_ERROR, std::string("no usable CUDA device (") + cudaGetErrorString(e) +
                                                   "); smgx has no CPU fallback — use device_id = -1 only for host-mirror tests");
            if (cfg.device_id >= count) throw Error(SMGX_INVALID_ARGUMENT, "device_id out of range");
            SMGX_CUDA(cudaSetDevice(cfg.device_id));
            cudaDeviceProp prop;
            SMGX_CUDA(cudaGetDeviceProperties(&prop, cfg.device_id));
            sm_count = prop.multiProcessorCount;
            l2_bytes = (size_t)prop.l2CacheSize;
            SMGX_CUDA(cudaStreamCreateWithFlags(&ctrl, cudaStreamNonBlocking));
            SMGX_CUDA(cudaEventCreateWithFlags(&state_ready, cudaEventDisableTiming));
            lanes.resize(4);
            for (auto& l : lanes) {
                SMGX_CUDA(cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking));
                SMGX_CUDA(cudaEventCreateWithFlags(&l.done, cudaEventDisableTiming));
                SMGX_CUDA(cudaEventCreate(&l.t0));
                SMGX_CUDA(cudaEventCreate(&l.t1));
                SMGX_CUDA(cudaStreamCreateWithFlags(&l.side, cudaStreamNonBlocking));
                SMGX_CUDA(cudaEventCreateWithFlags(&l.pre, cudaEventDisableTiming));
                SMGX_CUDA(cudaEventCreateWithFlags(&l.side_done, cudaEventDisableTiming));
                l.d_ready.reserve(kMaxMultiBatches * 4);
                SMGX_CUDA(cudaMemset(l.d_ready.ptr, 0, kMaxMultiBatches * 4));
            }
            d_err.reserve(64);
            SMGX_CUDA(cudaMemset(d_err.ptr, 0, 64));
            d_done_counters.reserve(kDoneCounters * 4);
            SMGX_CUDA(cudaMemset(d_done_counters.ptr, 0, kDoneCounters * 4));
        }
    }
    ~Policy() {
        stop_eviction_thread();
        if (cfg.device_id >= 0) {
            cudaSetDevice(cfg.device_id);
            cudaDeviceSynchronize();
            for (auto& l : lanes) {
                l.d_fb.release(); l.d_slowq.release(); l.d_recs.release(); l.d_groups.release(); l.d_tokens.release(); l.d_offsets.release(); l.d_out.release(); l.d_info.release(); l.d_hash.release();
                l.d_text.release(); l.d_toff.release(); l.d_path.release(); l.d_path_len.release(); l.d_tenant.release();
                l.d_path_tenant.release(); l.d_fill.release(); l.d_chunk_start.release(); l.d_cv.release(); l.d_hashes.release();
                l.tok_scratch.flags.release(); l.tok_scratch.tmp_ids.release(); l.tok_scratch.tmp_rk.release(); l.tok_scratch.totals.release();
                l.tok_scratch.pieces.release(); l.tok_scratch.n_pieces.release(); l.tok_scratch.miss.release();
                if (l.done) cudaEventDestroy(l.done);
                if (l.t0) cudaEventDestroy(l.t0);
                if (l.t1) cudaEventDestroy(l.t1);
                if (l.pre) cudaEventDestroy(l.pre);
                if (l.side_done) cudaEventDestroy(l.side_done);
                if (l.side) cudaStreamDestroy(l.side);
                l.d_ready.release();
                if (l.stream) cudaStreamDestroy(l.stream);
            }
            for (auto& kv : models) {
                ModelState& m = *kv.second;
                m.d_loads.release(); m.d_flags.release(); m.d_id_of_slice.release(); m.d_derived.release();
                m.d_slice_of_id.release(); m.d_load_of_id.release(); m.d_elig.release();
                m.indexer.reset();
                m.tokenizer.reset();
                m.token_tree.reset();
                m.string_tree.reset();
                m.d_slice_of_tenant.release();
                m.d_ring_pos.release(); m.d_ring_slice.release(); m.d_ring_url.release(); m.d_ring_bucket.release(); m.d_dup_prev.release();
                m.d_pf_loads.release(); m.d_pf_flags.release(); m.d_pf_derived.release(); m.d_ch_lists.release();
            }
            for (uint32_t i = 0; i < kPipeSlots; ++i) { if (pipe_hashed[i]) cudaEventDestroy(pipe_hashed[i]); if (pipe_searched[i]) cudaEventDestroy(pipe_searched[i]); }
            for (int b = 0; b < 2; ++b) {
                pf_hash_buf[b].release();
                if (pf_hash_ev[b]) cudaEventDestroy(pf_hash_ev[b]);
                if (pf_pick_ev[b]) cudaEventDestroy(pf_pick_ev[b]);
            }
            pf_stage.release(); pf_out.release(); pf_run_loads.release(); ch_stage.release(); ch_out.release();
            for (uint32_t q = 0; q < xch.peer.size(); ++q) if (q < xch.opened.size() && xch.opened[q] && xch.peer[q]) cudaIpcCloseMemHandle(xch.peer[q]);
            xch.local.release(); xch.d_bases.release(); xch.d_cand.release(); xch.d_fleet.release(); xch.d_arrive.release(); xch.d_gbase.release();
            d_err.release(); d_done_counters.release(); d_flush.release(); scratch.release(); scratch2.release(); d_gbase.release();
            if (state_ready) cudaEventDestroy(state_ready);
            if (ctrl) cudaStreamDestroy(ctrl);
        }
    }

    void use_device() const {
        if (cfg.device_id < 0)
            throw Error(SMGX_DEVICE_ERROR, "policy was created with device_id = -1 (host mirror only): no GPU path, no CPU fallback");
        SMGX_CUDA(cudaSetDevice(cfg.device_id));
    }

    ModelState& model(const char* key, bool create) {
        std::string k = norm_model(key);
        auto it = models.find(k);
        if (it != models.end()) return *it->second;
        if (!create) throw Error(SMGX_NOT_FOUND, "unknown model key '" + k + "'");
        auto& slot = models[k];
        slot = std::make_unique<ModelState>();
        return *slot;
    }
    EventIndex& indexer(const char* key) {
        ModelState& m = model(key, false);
        if (!m.indexer) throw Error(SMGX_NOT_FOUND, "no event indexer for model '" + norm_model(key) + "'");
        return *m.indexer;
    }

    // has_event_indexer (cache_aware.rs:723-729)
    bool has_event_indexer(const ModelState& m) const { return monitor && m.indexer && m.indexer->current_size() > 0; }
    uint32_t block_size_for(const ModelState& m) const { return m.has_learned_bs ? m.learned_bs : (uint32_t)cfg.block_size; }

    // Bring the device copies (index + fleet) up to date, in `ctrl` stream order, and make every lane wait for it.
    void sync_state(ModelState& m, EventIndexView* ixv, FleetView* fv) {
        uint64_t wv0 = m.indexer ? m.indexer->workers_version() : 0;
        bool pending = m.fleet_dirty || wv0 != m.seen_workers_version || (m.indexer && m.indexer->pending());
        // updates must not race with kernels still reading the previous state
        if (pending) for (auto& l : lanes) if (l.has_done) SMGX_CUDA(cudaStreamWaitEvent(ctrl, l.done, 0));
        EventIndexView v{};
        if (m.indexer) v = m.indexer->flush(ctrl, &launches);
        uint32_t n_ids = m.indexer ? m.indexer->n_workers() : 0;
        uint32_t words = m.indexer ? m.indexer->words() : 1;
        uint64_t wv = m.indexer ? m.indexer->workers_version() : 0;
        if (m.fleet_dirty || wv != m.seen_workers_version) {
            uint32_t ns = (uint32_t)m.urls.size();
            std::vector<int32_t> id_of_slice(std::max<uint32_t>(ns, 1), -1);
            for (uint32_t i = 0; i < ns; ++i) id_of_slice[i] = m.indexer ? (int32_t)m.indexer->worker_id(m.urls[i]) : -1;
            m.d_loads.reserve(std::max<uint32_t>(ns, 1) * 8);
            m.d_flags.reserve(std::max<uint32_t>(ns, 1));
            m.d_id_of_slice.reserve(std::max<uint32_t>(ns, 1) * 4);
            m.d_derived.reserve(sizeof(FleetDerived));
            m.d_slice_of_id.reserve(std::max<uint32_t>(n_ids, 1) * 4);
            m.d_load_of_id.reserve(std::max<uint32_t>(n_ids, 1) * 8);
            m.d_elig.reserve(kMaxWords * 8);
            if (ns) {
                SMGX_CUDA(cudaMemcpyAsync(m.d_loads.ptr, m.loads.data(), ns * 8, cudaMemcpyHostToDevice, ctrl));
                SMGX_CUDA(cudaMemcpyAsync(m.d_flags.ptr, m.flags.data(), ns, cudaMemcpyHostToDevice, ctrl));
                SMGX_CUDA(cudaMemcpyAsync(m.d_id_of_slice.ptr, id_of_slice.data(), ns * 4, cudaMemcpyHostToDevice, ctrl));
            }
            FleetRaw raw;
            raw.loads = m.d_loads.as<uint64_t>(); raw.flags = m.d_flags.as<uint8_t>(); raw.id_of_slice = m.d_id_of_slice.as<int32_t>();
            raw.n_slice = ns; raw.n_ids = n_ids; raw.words = words;
            raw.has_dups = 0;
            m.fleet_has_dups = false;
            {   // duplicate URLs in the slice → several slice entries share one indexer id
                std::vector<uint8_t> seen(std::max<uint32_t>(n_ids, 1), 0);
                for (uint32_t i = 0; i < ns; ++i) {
                    const int32_t id = id_of_slice[i];
                    if (id < 0 || (uint32_t)id >= n_ids) continue;
                    if (seen[(size_t)id]) { raw.has_dups = 1; m.fleet_has_dups = true; break; }
                    seen[(size_t)id] = 1;
                }
            }
            raw.abs_threshold = cfg.balance_abs_threshold; raw.rel_threshold = cfg.balance_rel_threshold;
            launch_fleet_prepare(raw, m.d_derived.as<FleetDerived>(), m.d_slice_of_id.as<int32_t>(), m.d_load_of_id.as<uint64_t>(),
                                 m.d_elig.as<uint64_t>(), ctrl);
            ++launches;
            m.fleet_dirty = false;
            m.seen_workers_version = wv;
        }
        if (pending) {
            SMGX_CUDA(cudaEventRecord(state_ready, ctrl));
            for (auto& l : lanes) SMGX_CUDA(cudaStreamWaitEvent(l.stream, state_ready, 0));
        }
        if (ixv) *ixv = v;
        if (fv) {
            fv->derived = m.d_derived.as<FleetDerived>();
            fv->slice_of_id = m.d_slice_of_id.as<int32_t>();
            fv->load_of_id = m.d_load_of_id.as<uint64_t>();
            fv->elig = m.d_elig.as<uint64_t>();
        }
    }

    static uint32_t max_n_of(const BatchDesc* d, uint32_t count) { uint32_t m = 0; for (uint32_t k = 0; k < count; ++k) m = std::max(m, d[k].n); return m; }
    // Enqueue the kernels of up to kMaxMultiBatches token batches on `lane` (device pointers).
    void enqueue_batches(ModelState& m, Lane& lane, const BatchDesc* descs, uint32_t count, uint32_t max_req_tokens, uint64_t* done_flag = nullptr,
                         uint64_t done_value = 0) {
        const bool cand_mode = count && descs[0].cand != nullptr;   // a worker-id shard may legitimately hold no blocks yet
        if (cand_mode && !m.indexer) throw Error(SMGX_NOT_FOUND, "no event indexer for this model");
        if (!cand_mode && !has_event_indexer(m))
            throw Error(SMGX_UNKNOWN_ERROR,
                        "model has no populated KV-event indexer: the approximate token-tree mode (cache_aware.rs:834-904) is not part of this "
                        "build yet — there is no CPU fallback");
        EventIndexView ixv;
        FleetView fv;
        sync_state(m, &ixv, &fv);
        uint32_t bs = block_size_for(m);
        MultiArgs a{};
        a.count = count;
        a.block_size = bs;
        a.max_blocks = bs ? std::max<uint32_t>(max_req_tokens / bs, 1) : 1;
        uint64_t rows = 0;
        bool uniform = true;
        for (uint32_t k = 0; k < count; ++k) { a.b[k] = descs[k]; a.b[k].hash_base = (uint32_t)rows; rows += descs[k].n; uniform = uniform && descs[k].n == descs[0].n; }
        SMGX_REQUIRE(rows < (1ull << 32), "too many requests in one launch");
        a.total = (uint32_t)rows;
        a.uniform_n = uniform && count ? descs[0].n : 0;
        a.hashes = nullptr;
        a.slow_queue = nullptr;
        if (event_select_fused() && !cand_mode && !done_flag && rows > 0) {   // queue of the simple kernel (zeroed when allocated; the slow kernel leaves the count and exit counter zeroed)
            const size_t need = ((size_t)rows + 2) * 4;
            if (need > lane.d_slowq.cap) {
                lane.d_slowq.reserve(need * 2);
                SMGX_CUDA(cudaMemsetAsync(lane.d_slowq.ptr, 0, lane.d_slowq.cap, lane.stream));
            }
            a.slow_queue = lane.d_slowq.as<uint32_t>();
            // a request is queued for event_slow_kernel only when it has more than 32 blocks, more than one jump, or meets a Multi entry:
            // with none of these possible (the multi count is the one of the view sync_state just flushed) the kernel is not launched
            a.skip_slow = m.indexer->multi_count() == 0 && a.max_blocks <= 32 && a.max_blocks - 1 <= ixv.jump;
        }
        a.fb_winsets = nullptr; a.fb_scores = nullptr;
        const bool feedback = load_feedback && !cand_mode && rows > 0;
        if (feedback) {
            if (m.fleet_has_dups) throw Error(SMGX_INVALID_ARGUMENT, "load feedback is not available for worker slices with duplicate URLs");
            lane.d_fb.reserve(rows * ixv.words * 8 + rows * 4 + 64);
            a.fb_winsets = lane.d_fb.as<uint64_t>();
            a.fb_scores = reinterpret_cast<uint32_t*>(lane.d_fb.as<uint64_t>() + rows * ixv.words);
        }
        a.done_flag = feedback ? nullptr : done_flag; a.done_value = done_value; a.done_counter = nullptr;
        if (feedback && done_flag) throw Error(SMGX_INVALID_ARGUMENT, "mapped submissions do not combine with load feedback (the in-order pass publishes the picks)");
        if (done_flag) {
            a.done_counter = d_done_counters.as<uint32_t>() + (done_seq++ % kDoneCounters);
        }
        a.pf_slots = nullptr; a.pf_mask = 0; a.pf_jump = 0; a.recs = nullptr; a.group_count = nullptr; a.group_stride = 0;
        { static const uint32_t dbg = [] { const char* e = getenv("SMGX_STREAM_DBG"); return e ? (uint32_t)atoi(e) : 0u; }(); a.dbg = dbg; }
        if (event_launch_is_split(a)) {
            if (&lane == &lanes[0])   // lane 0's scratch doubles as the ring of enqueue_split_pipelined: its readers run on lane 1
                for (uint32_t i = 0; i < kPipeSlots; ++i) if (pipe_used[i]) SMGX_CUDA(cudaStreamWaitEvent(lane.stream, pipe_searched[i], 0));
            lane.d_hash.reserve(std::max<uint64_t>(rows, 1) * a.max_blocks * 8);
            a.hashes = lane.d_hash.as<uint64_t>();
            lane.d_recs.reserve(std::max<uint64_t>(rows, 1) * sizeof(SearchRec));
            a.recs = lane.d_recs.as<SearchRec>();
            a.pf_slots = ixv.slots; a.pf_mask = ixv.mask; a.pf_jump = ixv.jump;
            if (event_path() == 2 && ixv.words == 1) {   // arrival counters of event_hs_kernel
                const uint32_t need = (max_n_of(descs, count) + 255) / 256;
                if (need > lane.group_stride) {
                    lane.group_stride = std::max<uint32_t>(need * 2, 64);
                    lane.d_groups.reserve((size_t)kMaxMultiBatches * lane.group_stride * 4);
                    SMGX_CUDA(cudaMemsetAsync(lane.d_groups.ptr, 0, (size_t)kMaxMultiBatches * lane.group_stride * 4, lane.stream));
                }
                a.group_count = lane.d_groups.as<uint32_t>(); a.group_stride = lane.group_stride;
            }
        }
        a.err_flag = d_err.as<uint32_t>();
        a.ready = nullptr;
        // concurrent split launch (SMGX_SPLIT_CONCURRENT=1, experiment): the search kernel starts together with the hash kernel on a side stream and
        // follows it batch by batch through device-side counters.  Measured worse than plain stream order (the waiting search
        // CTAs take registers from the hash stream and the stream join costs more than the overlap gains) — off by default.
        static const int concurrent = [] { const char* e = getenv("SMGX_SPLIT_CONCURRENT"); return e ? atoi(e) : 0; }();
        if (concurrent && event_launch_is_split(a) && ixv.words == 1 && count >= 2 && bs == 16 && (uint64_t)count * ((max_n_of(descs, count) + 255) / 256) <= (uint64_t)sm_count * 3) {
            const uint64_t threads = (uint64_t)max_n_of(descs, count) * a.max_blocks;
            const uint32_t gx = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((threads + 255) / 256, (uint64_t)sm_count * 64));   // = launch_event_hash's grid.x
            a.ready = lane.d_ready.as<uint32_t>();
            for (uint32_t k = 0; k < count; ++k) { lane.ready_cum[k] += gx; a.ready_target[k] = lane.ready_cum[k]; }
            SMGX_CUDA(cudaEventRecord(lane.pre, lane.stream));             // everything the kernels depend on (copies, state updates) is ordered before this
            SMGX_CUDA(cudaStreamWaitEvent(lane.side, lane.pre, 0));
            launch_event_hash(a, sm_count, lane.stream, &launches);
            launch_event_search(ixv, fv, a, sm_count, lane.side, &launches);
            SMGX_CUDA(cudaEventRecord(lane.side_done, lane.side));
            SMGX_CUDA(cudaStreamWaitEvent(lane.stream, lane.side_done, 0));  // the lane's later work (D2H of the picks, the next call's hash stream) follows the search
        } else
        launch_event_select(ixv, fv, a, sm_count, lane.stream, &launches);
        if (feedback) {
            launch_feedback_resolve(ixv, fv, a, m.d_loads.as<uint64_t>(), m.d_flags.as<uint8_t>(), (uint32_t)m.urls.size(), cfg.balance_abs_threshold,
                                    cfg.balance_rel_threshold, nullptr, lane.stream);
            ++launches;
        }
        SMGX_CUDA(cudaEventRecord(lane.done, lane.stream));
        lane.has_done = true;
    }
    // Several device-resident batches on the split path: the hash stream of chunk c+1 runs on lane 0 while the search of chunk c runs on
    // lane 1, so a call's duration is the hash stream (HBM-bound) plus the last chunk's search instead of the sum of both for every chunk.
    // The hash scratch is a ring of kPipeSlots chunk-sized regions guarded by events in both directions.
    static constexpr uint32_t kPipeSlots = 4;
    cudaEvent_t pipe_hashed[kPipeSlots] = {}, pipe_searched[kPipeSlots] = {};
    bool pipe_used[kPipeSlots] = {};
    uint64_t pipe_seq = 0;
    bool enqueue_split_pipelined(ModelState& m, const BatchDesc* descs, uint32_t count, uint32_t max_req_tokens) {
        // measured: the search kernel is a latency chain of about the same length whatever its size, so chunking a short call only
        // multiplies that chain — the two-lane pipeline stays opt-in (SMGX_SPLIT_PIPE=1) for experiments
        static const int pipe = [] { const char* e = getenv("SMGX_SPLIT_PIPE"); return e ? atoi(e) : 0; }();   // number of chunks a short call is cut into (0 = off)
        if (pipe < 2 || count < 2 || count > kMaxMultiBatches || lanes.size() < 4 || load_feedback || event_select_fused()) return false;
        if (!has_event_indexer(m)) return false;   // let enqueue_batches raise the error
        EventIndexView ixv;
        FleetView fv;
        sync_state(m, &ixv, &fv);
        const uint32_t bs = block_size_for(m);
        const uint32_t max_blocks = bs ? std::max<uint32_t>(max_req_tokens / bs, 1) : 1;
        // chunk size: at most kMaxMultiBatches, at least 2 chunks per call, about 4 for short calls so that only ~1/4 of the search is exposed
        const uint32_t per = std::min<uint32_t>(kMaxMultiBatches, std::max<uint32_t>(1, (count + (uint32_t)pipe - 1) / (uint32_t)pipe));
        uint32_t max_n = 0;
        for (uint32_t k = 0; k < count; ++k) max_n = std::max(max_n, descs[k].n);
        const uint64_t slot_rows = (uint64_t)per * max_n;
        SMGX_REQUIRE(slot_rows < (1ull << 32), "too many requests in one launch");
        Lane& lh = lanes[0];
        lh.d_hash.reserve(std::max<uint64_t>(slot_rows, 1) * max_blocks * 8 * kPipeSlots);
        for (uint32_t i = 0; i < kPipeSlots; ++i) if (!pipe_hashed[i]) {
            SMGX_CUDA(cudaEventCreateWithFlags(&pipe_hashed[i], cudaEventDisableTiming));
            SMGX_CUDA(cudaEventCreateWithFlags(&pipe_searched[i], cudaEventDisableTiming));
        }
        uint32_t chunk_idx = 0;
        for (uint32_t j0 = 0; j0 < count; j0 += per, ++chunk_idx) {
            const uint32_t cnt = std::min(per, count - j0);
            const uint32_t slot = (uint32_t)(pipe_seq++ % kPipeSlots);
            Lane& ls = lanes[1 + chunk_idx % 3];   // every chunk's search on its own lane: the searches are latency chains and must overlap each other too
            MultiArgs a{};
            a.count = cnt; a.block_size = bs; a.max_blocks = max_blocks;
            uint64_t rows = 0;
            bool uniform = true;
            for (uint32_t k = 0; k < cnt; ++k) { a.b[k] = descs[j0 + k]; a.b[k].hash_base = (uint32_t)rows; rows += descs[j0 + k].n; uniform = uniform && descs[j0 + k].n == descs[j0].n; }
            a.total = (uint32_t)rows; a.uniform_n = uniform ? descs[j0].n : 0;
            a.hashes = lh.d_hash.as<uint64_t>() + (uint64_t)slot * slot_rows * max_blocks;
            a.slow_queue = nullptr; a.fb_winsets = nullptr; a.fb_scores = nullptr;
            a.done_flag = nullptr; a.done_value = 0; a.done_counter = nullptr;
            a.pf_slots = ixv.slots; a.pf_mask = ixv.mask; a.pf_jump = ixv.jump;
            lh.d_recs.reserve(std::max<uint64_t>(slot_rows, 1) * sizeof(SearchRec) * kPipeSlots);
            a.recs = lh.d_recs.as<SearchRec>() + (uint64_t)slot * slot_rows;
            a.err_flag = d_err.as<uint32_t>();
            if (pipe_used[slot]) SMGX_CUDA(cudaStreamWaitEvent(lh.stream, pipe_searched[slot], 0));   // the region's previous reader is done
            launch_event_hash(a, sm_count, lh.stream, &launches);
            SMGX_CUDA(cudaEventRecord(pipe_hashed[slot], lh.stream));
            SMGX_CUDA(cudaStreamWaitEvent(ls.stream, pipe_hashed[slot], 0));
            launch_event_search(ixv, fv, a, sm_count, ls.stream, &launches);
            SMGX_CUDA(cudaEventRecord(pipe_searched[slot], ls.stream));
            pipe_used[slot] = true;
        }
        for (auto& l : lanes) { SMGX_CUDA(cudaEventRecord(l.done, l.stream)); l.has_done = true; }
        return true;
    }
    void enqueue_tokens(ModelState& m, Lane& lane, const uint32_t* d_tokens, const uint32_t* d_offsets, uint32_t n, uint32_t max_req_tokens,
                        int32_t* d_out, smgx_decision_info* d_info) {
        BatchDesc d{d_tokens, d_offsets, d_out, d_info, n, 0, nullptr};
        enqueue_batches(m, lane, &d, 1, max_req_tokens);
    }


    // hash_index.insert(hash, matched_prefix) (cache_aware.rs:881-886, :950-956) REPLACES the previous value.  Values live in one arena
    // per model: an existing key is overwritten in place when the new prefix fits, otherwise the old bytes are counted dead and the
    // arena is compacted once more than half of it is dead — repeated identical requests no longer grow it.
    static void hash_index_put_tokens(ModelState& m, uint64_t key, const uint32_t* tk, uint32_t len) {
        auto it = m.hash_index_tokens.find(key);
        if (it != m.hash_index_tokens.end()) {
            if (len <= it->second.second) {
                std::copy(tk, tk + len, m.hash_arena_tokens.begin() + (ptrdiff_t)it->second.first);
                m.hash_dead_tokens += it->second.second - len;
                it->second.second = len;
                return;
            }
            m.hash_dead_tokens += it->second.second;
        }
        m.hash_index_tokens[key] = {m.hash_arena_tokens.size(), len};
        m.hash_arena_tokens.insert(m.hash_arena_tokens.end(), tk, tk + len);
        if (m.hash_dead_tokens > 4096 && m.hash_dead_tokens * 2 > m.hash_arena_tokens.size()) {
            std::vector<uint32_t> live;
            live.reserve(m.hash_arena_tokens.size() - m.hash_dead_tokens);
            for (auto& kv : m.hash_index_tokens) {
                const uint64_t at = live.size();
                live.insert(live.end(), m.hash_arena_tokens.begin() + (ptrdiff_t)kv.second.first, m.hash_arena_tokens.begin() + (ptrdiff_t)(kv.second.first + kv.second.second));
                kv.second.first = at;
            }
            m.hash_arena_tokens.swap(live);
            m.hash_dead_tokens = 0;
        }
    }
    static void hash_index_put_text(ModelState& m, uint64_t key, const uint8_t* tx, uint32_t len) {
        auto it = m.hash_index_text.find(key);
        if (it != m.hash_index_text.end()) {
            if (len <= it->second.second) {
                memcpy(&m.hash_arena_text[(size_t)it->second.first], tx, len);
                m.hash_dead_text += it->second.second - len;
                it->second.second = len;
                return;
            }
            m.hash_dead_text += it->second.second;
        }
        m.hash_index_text[key] = {m.hash_arena_text.size(), len};
        m.hash_arena_text.append((const char*)tx, len);
        if (m.hash_dead_text > 16384 && m.hash_dead_text * 2 > m.hash_arena_text.size()) {
            std::string live;
            live.reserve(m.hash_arena_text.size() - m.hash_dead_text);
            for (auto& kv : m.hash_index_text) {
                const uint64_t at = live.size();
                live.append(m.hash_arena_text, (size_t)kv.second.first, kv.second.second);
                kv.second.first = at;
            }
            m.hash_arena_text.swap(live);
            m.hash_dead_text = 0;
        }
    }

    TokenTreeIndex& tree_of(ModelState& m, bool create) {
        if (!m.token_tree) {
            if (!create) throw Error(SMGX_NOT_FOUND, "no token tree for this model (call smgx_set_workers first)");
            m.token_tree = std::make_unique<TokenTreeIndex>(&tenants, &token_ts, EVP_LRU);
            m.token_tree->device_enabled = cfg.device_id >= 0;
        }
        return *m.token_tree;
    }
    // fleet-side lookup the tree pick needs: tenant id → first slice index with that URL (`position(|w| w.url() == tenant)`)
    void sync_tenant_map(ModelState& m) {
        if (!m.fleet_dirty_tenant && m.seen_tenants_version == tenants.version) return;
        m.tenant_of_slice.resize(m.urls.size());
        for (size_t i = 0; i < m.urls.size(); ++i) m.tenant_of_slice[i] = tenants.intern(m.urls[i]);   // the inverse, for the insert's tenant
        std::vector<int32_t> sl(std::max<size_t>(tenants.names.size(), 1), -1);
        for (size_t i = m.urls.size(); i-- > 0;) {
            int64_t t = tenants.find(m.urls[i]);
            if (t >= 0) sl[(size_t)t] = (int32_t)i;   // iterating downwards leaves the FIRST position
        }
        m.d_slice_of_tenant.reserve(sl.size() * 4);
        SMGX_CUDA(cudaMemcpyAsync(m.d_slice_of_tenant.ptr, sl.data(), sl.size() * 4, cudaMemcpyHostToDevice, ctrl));
        SMGX_CUDA(cudaStreamSynchronize(ctrl));
        m.slice_of_tenant.swap(sl);
        m.fleet_dirty_tenant = false;
        m.seen_tenants_version = tenants.version;
    }
    // the f32 imbalance gate of fleet_prepare_kernel (cache_aware.rs:669-670): round-to-nearest conversions, an f32 product, strict >
    bool imbalanced_f32(uint64_t mn, uint64_t mx) const {
        volatile float fmax = (float)mx;
        volatile float fprod = (float)mn * cfg.balance_rel_threshold;
        return (mx - mn) > cfg.balance_abs_threshold && fmax > fprod;
    }
    bool host_imbalanced(const ModelState& m) const {   // used for mode dispatch only
        if (m.loads.empty()) return false;
        uint64_t mn = ~0ULL, mx = 0;
        for (uint64_t l : m.loads) { mn = std::min(mn, l); mx = std::max(mx, l); }
        return imbalanced_f32(mn, mx);
    }

    // The fleet a tree-mode load-feedback batch runs against: the snapshot loads plus one per pick so far (the router's WorkerLoadGuard,
    // routers/http/router.rs:319-321).  Kept as feedback_resolve_kernel keeps it: min / max over ALL workers (cache_aware.rs:662-666) with
    // the number of workers at the minimum, and the first argmin over healthy workers with an ok circuit (min_by_key → FIRST minimum),
    // looked for again only after it was itself picked.  The tree modes decide on the host, in the in-order pass that already commits
    // every request's side effects, so a bump costs no launch.
    struct RunningFleet {
        std::vector<uint64_t> load;
        const uint8_t* flags;
        uint64_t gmin = ~0ULL, gmax = 0;
        uint32_t at_gmin = 0;
        int32_t hidx = -1, first_healthy = -1;
        explicit RunningFleet(const ModelState& m) : load(m.loads), flags(m.flags.data()) {
            for (size_t i = 0; i < load.size(); ++i) {
                gmin = std::min(gmin, load[i]);
                gmax = std::max(gmax, load[i]);
                if (first_healthy < 0 && (flags[i] & 3) == 3) first_healthy = (int32_t)i;
            }
            if (load.empty()) gmin = 0;
            for (uint64_t l : load) at_gmin += l == gmin;
            rescan();
        }
        void rescan() {
            hidx = -1;
            for (size_t i = 0; i < load.size(); ++i)
                if ((flags[i] & 3) == 3 && (hidx < 0 || load[i] < load[(size_t)hidx])) hidx = (int32_t)i;
        }
        void bump(int32_t w) {
            const uint64_t old = load[(size_t)w]++;
            gmax = std::max(gmax, old + 1);
            if (old == gmin && --at_gmin == 0) { ++gmin; for (uint64_t l : load) at_gmin += l == gmin; }
            if (w != hidx) return;
            // workers before hidx are above the old minimum: the next argmin is a later worker still at it, or else found by a rescan
            for (size_t i = (size_t)w + 1; i < load.size(); ++i)
                if ((flags[i] & 3) == 3 && load[i] == old) { hidx = (int32_t)i; return; }
            rescan();
        }
    };
    // select_worker's load-dependent decision for one walked request against the running fleet (SURVEY Appendix A.1 steps 3, 4, 6/7):
    // gate open → the first healthy argmin (select_worker_min_load); match rate above the threshold → the tenant's first slice position if
    // is_healthy(), else healthy[0] (:892-894); otherwise the first healthy argmin.  Same f32 arithmetic as tree_walk_request.
    void decide_running(const ModelState& m, const RunningFleet& rf, uint32_t matched, uint32_t input, int32_t tenant, int32_t* out,
                        uint8_t* branch) const {
        if (imbalanced_f32(rf.gmin, rf.gmax)) { *out = rf.hidx; *branch = SMGX_BR_IMBALANCED_MIN_LOAD; return; }
        volatile float rate = input == 0 ? 0.0f : (float)matched / (float)input;
        if (rate > cfg.cache_threshold) {
            const int32_t sl = (tenant >= 0 && (size_t)tenant < m.slice_of_tenant.size()) ? m.slice_of_tenant[(size_t)tenant] : -1;
            if (sl >= 0 && (m.flags[(size_t)sl] & 1)) { *out = sl; *branch = SMGX_BR_TREE_MATCH; }
            else { *out = rf.first_healthy; *branch = SMGX_BR_TREE_FALLBACK_FIRST_HEALTHY; }
        } else { *out = rf.hidx; *branch = SMGX_BR_TREE_MIN_LOAD; }
    }
    void refuse_snapshot_feedback() const {
        if (tree_feedback && tree_batch_mode == SMGX_TREE_BATCH_SNAPSHOT)
            throw Error(SMGX_INVALID_ARGUMENT, "cache_aware load feedback does not combine with SMGX_TREE_BATCH_SNAPSHOT (use SEQUENTIAL)");
    }

    // Approximate-token-tree mode (cache_aware.rs:834-904) and the imbalanced path's tree update (:380-402).
    // SMGX_TREE_BATCH_SEQUENTIAL: requests are processed in contiguous segments whose first-page keys are pairwise distinct:
    // such requests touch disjoint subtrees, so matching a whole segment against one snapshot on the GPU and then applying
    // touches + inserts on the host in request order reproduces the reference's one-by-one semantics exactly (timestamps
    // included).  SMGX_TREE_BATCH_SNAPSHOT: the whole batch is one segment — every request walks and decides against the
    // pre-batch tree, then the side effects are applied in request order: one admissible interleaving of concurrent
    // select_worker calls (include/smgx.h), identical to SEQUENTIAL when no two requests of the batch share a first page.
    // `forced` (load-feedback mode): the picks were made by the in-order pass; this call only performs select_worker_min_load's tree side
    // effects (match touches, insert under the picked worker, hash_index; cache_aware.rs:380-402) for them.  `use_lane`: whose staging and
    // stream to use (default lane 0).
    void tree_select(ModelState& m, const uint32_t* tokens, const uint32_t* offsets, uint32_t n, int32_t* out_idx, smgx_decision_info* out_info,
                     bool decide, int32_t* out_tenant, const int32_t* forced = nullptr, Lane* use_lane = nullptr) {
        TokenTreeIndex& tree = tree_of(m, true);
        Lane& lane = use_lane ? *use_lane : lanes[0];
        if (forced) decide = false;
        if (decide) refuse_snapshot_feedback();
        const uint64_t base = n ? offsets[0] : 0, total = n ? offsets[n] - base : 0;
        const uint32_t n1 = std::max<uint32_t>(n, 1);
        lane.d_tokens.reserve(std::max<uint64_t>(total, 1) * 4 + 16);
        lane.d_offsets.reserve(((size_t)n + 1) * 4);
        lane.d_out.reserve(n1 * 4);
        lane.d_info.reserve(n1 * sizeof(smgx_decision_info));
        lane.d_path.reserve((size_t)n1 * kPathCap * 4);
        lane.d_path_tenant.reserve((size_t)n1 * kPathCap * 4);
        lane.d_path_len.reserve(n1 * 4);
        lane.d_tenant.reserve(n1 * 4);
        if (n == 0) return;
        if (total) SMGX_CUDA(cudaMemcpyAsync(lane.d_tokens.ptr, tokens + base, total * 4, cudaMemcpyHostToDevice, lane.stream));
        SMGX_CUDA(cudaMemcpyAsync(lane.d_offsets.ptr, offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, lane.stream));
        std::vector<smgx_decision_info> info(n);
        std::vector<uint32_t> path((size_t)n * kPathCap), path_len(n);
        std::vector<int32_t> path_ten((size_t)n * kPathCap), ten(n);
        std::vector<uint64_t> path_hash;   // hash_token_path of every request, for the hash_index side effect (:881-886, :397-401)
        if (decide || forced) enqueue_path_hashes(lane, reinterpret_cast<const uint8_t*>(lane.d_tokens.as<uint32_t>() - base), lane.d_offsets.as<uint32_t>(), offsets, n, 4, path_hash);
        const bool snapshot = tree_batch_mode == SMGX_TREE_BATCH_SNAPSHOT;
        // SEQUENTIAL is run optimistically: the rest of the batch is walked against one snapshot, then the host replays the
        // requests in order and stops at the first one whose snapshot walk is no longer what a walk at that moment would
        // return — a path node was split, the node the walk stopped under gained a child for the next page, or (when the pick
        // used it) the deepest node's tenant changed.  Everything before it is committed; the walk restarts from there.
        // Load feedback: the kernel's decision read the snapshot loads; each request is decided again here, in order, against the running
        // fleet, which carries the committed prefix's bumps across restarts.
        std::unique_ptr<RunningFleet> rf;
        if (decide && tree_feedback) rf = std::make_unique<RunningFleet>(m);
        uint32_t seg = 0;
        while (seg < n) {
            const uint32_t end = n;
            EventIndexView ixv;
            FleetView fv;
            sync_state(m, &ixv, &fv);
            sync_tenant_map(m);
            TokenTreeView tv = tree.flush(lane.stream, &launches);
            TreeSelectArgs a;
            a.tokens = lane.d_tokens.as<uint32_t>() - base; a.offsets = lane.d_offsets.as<uint32_t>();
            a.first = seg; a.count = end - seg;
            a.out_idx = lane.d_out.as<int32_t>(); a.out_info = lane.d_info.as<smgx_decision_info>();
            a.out_path = lane.d_path.as<uint32_t>(); a.out_path_tenant = lane.d_path_tenant.as<int32_t>();
            a.out_path_len = lane.d_path_len.as<uint32_t>(); a.out_tenant = lane.d_tenant.as<int32_t>();
            a.cache_threshold = cfg.cache_threshold; a.decide = decide ? 1 : 0;
            launch_tree_select(tv, fv, m.d_slice_of_tenant.as<int32_t>(), m.d_flags.as<uint8_t>(), (uint32_t)tenants.names.size(), a, lane.stream);
            ++launches;
            const uint32_t cnt = end - seg;
            SMGX_CUDA(cudaMemcpyAsync(out_idx + seg, lane.d_out.as<int32_t>() + seg, (size_t)cnt * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(info.data() + seg, lane.d_info.as<smgx_decision_info>() + seg, (size_t)cnt * sizeof(smgx_decision_info), cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(path.data() + (size_t)seg * kPathCap, lane.d_path.as<uint32_t>() + (size_t)seg * kPathCap, (size_t)cnt * kPathCap * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(path_ten.data() + (size_t)seg * kPathCap, lane.d_path_tenant.as<int32_t>() + (size_t)seg * kPathCap, (size_t)cnt * kPathCap * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(path_len.data() + seg, lane.d_path_len.as<uint32_t>() + seg, (size_t)cnt * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(ten.data() + seg, lane.d_tenant.as<int32_t>() + seg, (size_t)cnt * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaStreamSynchronize(lane.stream));
            tree.begin_chunk();
            // walks deeper than the kernel reports: recover the node list from the same (still unmodified) tree state
            std::unordered_map<uint32_t, TreeMatch> deep;
            if (snapshot)
                for (uint32_t r = seg; r < end; ++r)
                    if (path_len[r] > kPathCap) deep.emplace(r, tree.match_prefix_host(tokens + offsets[r], offsets[r + 1] - offsets[r], false));
            uint32_t r = seg;
            for (; r < end; ++r) {
                const uint32_t* tk = tokens + offsets[r];
                const uint32_t len = offsets[r + 1] - offsets[r];
                if (decide && info[r].branch == SMGX_BR_NO_HEALTHY) continue;   // returns None before touching anything (:653-655)
                int32_t pick = out_idx[r];
                uint8_t pick_br = info[r].branch;
                if (rf) decide_running(m, *rf, info[r].matched, info[r].input, ten[r], &pick, &pick_br);
                const uint32_t* pth = path.data() + (size_t)r * kPathCap;
                if (!snapshot && r > seg) {   // is the snapshot walk still the walk the reference would do now?
                    bool valid = path_len[r] <= kPathCap;
                    uint64_t sum_len = 0;
                    for (uint32_t d = 0; valid && d < path_len[r]; ++d) { valid = !tree.split_in_chunk(pth[d]); sum_len += tree.label_len_of(pth[d]); }
                    const uint8_t br = pick_br;
                    if (valid && path_len[r] && (br == SMGX_BR_TREE_MATCH || br == SMGX_BR_TREE_FALLBACK_FIRST_HEALTHY))
                        valid = tree.any_tenant(pth[path_len[r] - 1]) == ten[r];                       // the pick read this tenant
                    const uint32_t aligned = (len / kPage) * kPage;
                    if (valid && sum_len == info[r].matched && aligned - info[r].matched >= kPage)     // stopped under a node: still no child for the next page?
                        valid = !tree.has_child(path_len[r] ? pth[path_len[r] - 1] : 0, tk + info[r].matched);
                    if (!valid) break;
                }
                // match side effects: touch_tenant on every matched node, in order (:685-689)
                if (snapshot) {
                    if (path_len[r] <= kPathCap) tree.apply_match_touches(pth, path_ten.data() + (size_t)r * kPathCap, path_len[r]);
                    else { const TreeMatch& hm = deep.at(r); tree.apply_match_touches(hm.path.data(), hm.path_tenants.data(), (uint32_t)hm.path.size()); }
                } else if (path_len[r] <= kPathCap) tree.apply_match_touches(pth, path_len[r]);        // tenants as they are now
                else { TreeMatch hm = tree.match_prefix_host(tk, len, false); tree.apply_match_touches(hm.path.data(), (uint32_t)hm.path.size()); }
                if (forced) {
                    if (forced[r] >= 0 && (size_t)forced[r] < m.tenant_of_slice.size()) {
                        tree.insert_tokens(tk, len, m.tenant_of_slice[(size_t)forced[r]]);   // :396
                        hash_index_put_tokens(m, path_hash[r], tk, info[r].matched);
                    }
                    continue;
                }
                if (!decide) continue;
                if (rf) {
                    out_idx[r] = pick; info[r].branch = pick_br;
                    if (pick >= 0) rf->bump(pick);   // WorkerLoadGuard on whatever select_worker returned, healthy[0] included
                }
                const uint8_t br = info[r].branch;
                if ((br == SMGX_BR_TREE_MATCH || br == SMGX_BR_TREE_MIN_LOAD || br == SMGX_BR_IMBALANCED_MIN_LOAD) && out_idx[r] >= 0) {
                    const size_t idx = (size_t)out_idx[r];
                    tree.insert_tokens(tk, len, m.tenant_of_slice[idx]);   // :868 / :396
                    hash_index_put_tokens(m, path_hash[r], tk, info[r].matched);
                    if (idx < m.processed.size()) ++m.processed[idx];
                }
            }
            seg = r;
        }
        if (out_info) memcpy(out_info, info.data(), (size_t)n * sizeof(smgx_decision_info));
        if (out_tenant) memcpy(out_tenant, ten.data(), (size_t)n * 4);
    }

    // smg_mesh::hash_token_path / hash_node_path (crates/mesh/src/hash.rs:22-52) of every request of a batch that is already
    // on the device: enqueues the blake3 kernels and the copy back on `lane`; `out` is valid after the next stream sync.
    void enqueue_path_hashes(Lane& lane, const uint8_t* d_data, const uint32_t* d_offsets, const uint32_t* offsets, uint32_t n, uint32_t elem_bytes,
                             std::vector<uint64_t>& out, bool remap_zero = true) {
        out.assign(n, 0);
        if (n == 0) return;
        std::vector<uint32_t> chunk_start(n + 1);
        uint64_t total = 0;
        for (uint32_t i = 0; i < n; ++i) {
            chunk_start[i] = (uint32_t)total;
            const uint64_t bytes = (uint64_t)(offsets[i + 1] - offsets[i]) * elem_bytes;
            total += std::max<uint64_t>(1, (bytes + 1023) / 1024);
        }
        SMGX_REQUIRE(total < (1ull << 32), "too many blake3 chunks in one batch");
        chunk_start[n] = (uint32_t)total;
        lane.d_chunk_start.reserve(((size_t)n + 1) * 4);
        lane.d_cv.reserve((size_t)total * 32);
        lane.d_hashes.reserve((size_t)n * 8);
        SMGX_CUDA(cudaMemcpyAsync(lane.d_chunk_start.ptr, chunk_start.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, lane.stream));
        launch_blake3_paths(d_data, d_offsets, elem_bytes, lane.d_chunk_start.as<uint32_t>(), n, (uint32_t)total, lane.d_cv.as<uint32_t>(),
                            lane.d_hashes.as<uint64_t>(), lane.stream, &launches, remap_zero);
        SMGX_CUDA(cudaMemcpyAsync(out.data(), lane.d_hashes.ptr, (size_t)n * 8, cudaMemcpyDeviceToHost, lane.stream));
    }

    // ---- prefix_hash policy ----
    // blake3(bytes)[..8] (LE) of n byte strings, on the GPU: ring positions of virtual nodes and of routing keys (hash_ring.rs:78-86)
    void ring_positions(const std::string& blob, const std::vector<uint32_t>& offs, std::vector<uint64_t>& out) {
        const uint32_t n = (uint32_t)offs.size() - 1;
        out.assign(n, 0);
        if (n == 0) return;
        Lane& lane = lanes[0];
        lane.d_text.reserve(std::max<size_t>(blob.size(), 1) + 16);
        lane.d_offsets.reserve(((size_t)n + 1) * 4);
        if (!blob.empty()) SMGX_CUDA(cudaMemcpyAsync(lane.d_text.ptr, blob.data(), blob.size(), cudaMemcpyHostToDevice, lane.stream));
        SMGX_CUDA(cudaMemcpyAsync(lane.d_offsets.ptr, offs.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, lane.stream));
        enqueue_path_hashes(lane, lane.d_text.as<uint8_t>(), lane.d_offsets.as<uint32_t>(), offs.data(), n, 1, out, false);
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
    }
    // HashRing::new (hash_ring.rs:45-70)
    void ring_set(ModelState& m, const char* const* urls, uint32_t n) {
        std::string blob;
        std::vector<uint32_t> offs{0};
        for (uint32_t u = 0; u < n; ++u)
            for (uint32_t v = 0; v < kVirtualNodesPerWorker; ++v) {
                blob += urls[u]; blob += '#'; blob += std::to_string(v);   // format!("{url}#{vnode}")
                SMGX_REQUIRE(blob.size() < (1ull << 32), "ring too large");
                offs.push_back((uint32_t)blob.size());
            }
        std::vector<uint64_t> pos;
        ring_positions(blob, offs, pos);
        std::vector<uint32_t> order(pos.size());
        for (uint32_t i = 0; i < order.size(); ++i) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return pos[a] < pos[b]; });
        m.ring_urls.clear();
        for (uint32_t u = 0; u < n; ++u) m.ring_urls.emplace_back(urls[u]);
        m.ring_pos.resize(order.size());
        m.ring_url.resize(order.size());
        for (uint32_t i = 0; i < order.size(); ++i) { m.ring_pos[i] = pos[order[i]]; m.ring_url[i] = order[i] / kVirtualNodesPerWorker; }
        m.has_ring = true;
        m.pf_struct_dirty = true;
    }
    // device copies for the prefix_hash kernels, in lane-0 stream order
    void sync_prefix(ModelState& m, RingView* rv, PrefixFleetView* fv) {
        Lane& lane = lanes[0];
        const uint32_t ns = (uint32_t)m.urls.size(), len = m.has_ring ? (uint32_t)m.ring_pos.size() : 0;
        if (m.pf_struct_dirty || m.pf_state_dirty)   // pick kernels still running on the side lane read the arrays about to be replaced
            for (int b = 0; b < 2; ++b) if (pf_pick_pending[b]) SMGX_CUDA(cudaStreamWaitEvent(lane.stream, pf_pick_ev[b], 0));
        if (m.pf_struct_dirty) {
            // `healthy_url_map` (prefix_hash.rs:155-159) collects url → (idx, worker) over the healthy workers in slice order, later
            // duplicates overwriting earlier ones: a ring URL resolves to the LAST healthy slice index carrying it.  last_of / dup_prev
            // give the kernel that chain without knowing the health flags.
            std::unordered_map<std::string, int32_t> last_of;
            std::vector<int32_t> dup_prev(std::max<uint32_t>(ns, 1), -1);
            for (uint32_t i = 0; i < ns; ++i) {
                auto it = last_of.find(m.urls[i]);
                if (it != last_of.end()) { dup_prev[i] = it->second; it->second = (int32_t)i; }
                else last_of.emplace(m.urls[i], (int32_t)i);
            }
            std::vector<int32_t> slice_of_url(std::max<size_t>(m.ring_urls.size(), 1), -1), ring_slice(std::max<uint32_t>(len, 1), -1);
            for (size_t u = 0; u < m.ring_urls.size(); ++u) { auto it = last_of.find(m.ring_urls[u]); if (it != last_of.end()) slice_of_url[u] = it->second; }
            for (uint32_t e = 0; e < len; ++e) ring_slice[e] = slice_of_url[m.ring_url[e]];
            uint32_t kbits = 1;
            while ((1ull << kbits) < 2ull * len && kbits < 31) ++kbits;
            const uint32_t nbk = 1u << kbits;
            std::vector<uint32_t> bucket(nbk + 1);
            for (uint32_t b = 0, e = 0; b <= nbk; ++b) {
                if (b == nbk) { bucket[b] = len; break; }
                const uint64_t lower = (uint64_t)b << (64 - kbits);
                while (e < len && m.ring_pos[e] < lower) ++e;
                bucket[b] = e;
            }
            m.ring_bucket_shift = 64 - kbits;
            m.d_ring_bucket.reserve(bucket.size() * 4);
            SMGX_CUDA(cudaMemcpyAsync(m.d_ring_bucket.ptr, bucket.data(), bucket.size() * 4, cudaMemcpyHostToDevice, lane.stream));
            m.d_ring_pos.reserve(std::max<uint32_t>(len, 1) * 8);
            m.d_ring_slice.reserve(std::max<uint32_t>(len, 1) * 4);
            m.d_ring_url.reserve(std::max<uint32_t>(len, 1) * 4);
            m.d_dup_prev.reserve(std::max<uint32_t>(ns, 1) * 4);
            if (len) {
                SMGX_CUDA(cudaMemcpyAsync(m.d_ring_pos.ptr, m.ring_pos.data(), (size_t)len * 8, cudaMemcpyHostToDevice, lane.stream));
                SMGX_CUDA(cudaMemcpyAsync(m.d_ring_slice.ptr, ring_slice.data(), (size_t)len * 4, cudaMemcpyHostToDevice, lane.stream));
                SMGX_CUDA(cudaMemcpyAsync(m.d_ring_url.ptr, m.ring_url.data(), (size_t)len * 4, cudaMemcpyHostToDevice, lane.stream));
            }
            if (ns) SMGX_CUDA(cudaMemcpyAsync(m.d_dup_prev.ptr, dup_prev.data(), (size_t)ns * 4, cudaMemcpyHostToDevice, lane.stream));
            SMGX_CUDA(cudaStreamSynchronize(lane.stream));   // the staging vectors die here
            m.pf_struct_dirty = false;
            m.pf_state_dirty = true;
        }
        if (m.pf_state_dirty) {
            m.d_pf_loads.reserve(std::max<uint32_t>(ns, 1) * 8);
            m.d_pf_flags.reserve(std::max<uint32_t>(ns, 1));
            m.d_pf_derived.reserve(sizeof(PrefixDerived));
            if (ns) {
                SMGX_CUDA(cudaMemcpyAsync(m.d_pf_loads.ptr, m.loads.data(), (size_t)ns * 8, cudaMemcpyHostToDevice, lane.stream));
                SMGX_CUDA(cudaMemcpyAsync(m.d_pf_flags.ptr, m.flags.data(), ns, cudaMemcpyHostToDevice, lane.stream));   // pageable source: staged before return
            }
            launch_prefix_fleet_prepare(m.d_pf_loads.as<uint64_t>(), m.d_pf_flags.as<uint8_t>(), ns, prefix_load_factor, m.d_pf_derived.as<PrefixDerived>(),
                                        lane.stream);
            ++launches;
            m.pf_state_dirty = false;
            m.ch_dirty = true;
        }
        rv->pos = m.d_ring_pos.as<uint64_t>(); rv->slice = m.d_ring_slice.as<int32_t>(); rv->len = len; rv->has_ring = m.has_ring ? 1u : 0u;
        rv->bucket = m.d_ring_bucket.as<uint32_t>(); rv->bucket_shift = m.ring_bucket_shift;
        fv->loads = m.d_pf_loads.as<uint64_t>(); fv->flags = m.d_pf_flags.as<uint8_t>(); fv->dup_prev = m.d_dup_prev.as<int32_t>();
        fv->derived = m.d_pf_derived.as<PrefixDerived>(); fv->n_slice = ns;
    }
    // ring and fleet views for consistent_hashing, with the two index lists of the current fleet snapshot (in lane-0 stream order)
    void sync_chash(ModelState& m, RingView* rv, PrefixFleetView* fv) {
        sync_prefix(m, rv, fv);
        if (!m.ch_dirty) return;
        const uint32_t ns = (uint32_t)m.urls.size();
        m.ch_lists.clear();
        std::unordered_map<std::string, int32_t> last_of;   // healthy_url_to_idx (consistent_hashing.rs:74-79): a later duplicate overwrites
        for (uint32_t i = 0; i < ns; ++i)
            if (m.flags[i] & 1) { m.ch_lists.push_back((int32_t)i); last_of[m.urls[i]] = (int32_t)i; }
        m.ch_n_healthy = (uint32_t)m.ch_lists.size();
        for (auto& kv : last_of) m.ch_lists.push_back(kv.second);
        std::sort(m.ch_lists.begin() + m.ch_n_healthy, m.ch_lists.end());   // sort_unstable (:95)
        m.d_ch_lists.reserve(std::max<size_t>(m.ch_lists.size(), 1) * 4);
        Lane& lane = lanes[0];
        if (!m.ch_lists.empty())
            SMGX_CUDA(cudaMemcpyAsync(m.d_ch_lists.ptr, m.ch_lists.data(), m.ch_lists.size() * 4, cudaMemcpyHostToDevice, lane.stream));
        m.ch_dirty = false;
    }
    PinBuf ch_stage, ch_out;             // pinned staging of the consistent_hashing call
    uint64_t prefix_token_count = 256;   // PrefixHashConfig::default() (prefix_hash.rs:52-58)
    double prefix_load_factor = 1.25;
    PinBuf pf_stage, pf_out;             // pinned staging of the host-buffer prefix_hash call
    // power_of_two policy (policies/power_of_two.rs:22): cached_loads, reduced to what select_worker reads — effective_token_usage() per URL
    std::unordered_map<std::string, double> p2c_usage;
    DevBuf pf_hash_buf[2];               // prefix hashes between the hash and pick kernels of the device-resident path
    DevBuf pf_run_loads;                 // load feedback: running loads carried from one launch of a device-resident call to the next
    cudaEvent_t pf_hash_ev[2] = {nullptr, nullptr}, pf_pick_ev[2] = {nullptr, nullptr};
    bool pf_pick_pending[2] = {false, false};
    uint64_t pf_group = 0;

    StringTreeIndex& stree_of(ModelState& m) {
        if (!m.string_tree) {
            m.string_tree = std::make_unique<StringTreeIndex>(&tenants, &string_epoch);
            m.string_tree->device_enabled = cfg.device_id >= 0;
        }
        return *m.string_tree;
    }

    // HTTP text mode (select_worker_with_text, cache_aware.rs:907-974, and the imbalanced path's tree update :403-425) on the
    // char-level string tree.  Same batching contract as tree_select; in SEQUENTIAL mode two requests conflict when they
    // start with the same char under the root (they then share a subtree) or when both end on the root itself.
    void text_select(ModelState& m, const uint8_t* text, const uint32_t* offsets, uint32_t n, int32_t* out_idx, smgx_decision_info* out_info,
                     bool decide, int32_t* out_tenant) {
        if (decide) refuse_snapshot_feedback();
        StringTreeIndex& tree = stree_of(m);
        Lane& lane = lanes[0];
        const uint64_t base = n ? offsets[0] : 0, total = n ? offsets[n] - base : 0;
        const uint32_t n1 = std::max<uint32_t>(n, 1);
        lane.d_text.reserve(std::max<uint64_t>(total, 1) + 16);
        lane.d_offsets.reserve(((size_t)n + 1) * 4);
        lane.d_out.reserve(n1 * 4);
        lane.d_info.reserve(n1 * sizeof(smgx_decision_info));
        lane.d_path_len.reserve(n1 * 4);
        lane.d_tenant.reserve(n1 * 4);
        lane.d_fill.reserve(n1);
        if (n == 0) return;
        if (total) SMGX_CUDA(cudaMemcpyAsync(lane.d_text.ptr, text + base, total, cudaMemcpyHostToDevice, lane.stream));
        SMGX_CUDA(cudaMemcpyAsync(lane.d_offsets.ptr, offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, lane.stream));
        std::vector<smgx_decision_info> info(n);
        std::vector<uint32_t> node(n);
        std::vector<int32_t> ten(n);
        std::vector<uint8_t> fill(n);
        std::vector<uint64_t> path_hash;   // hash_node_path of every request (:950-956, :420-424)
        if (decide) enqueue_path_hashes(lane, lane.d_text.as<uint8_t>() - base, lane.d_offsets.as<uint32_t>(), offsets, n, 1, path_hash);
        const bool snapshot = tree_batch_mode == SMGX_TREE_BATCH_SNAPSHOT;
        std::unique_ptr<RunningFleet> rf;   // load feedback, as in tree_select
        if (decide && tree_feedback) rf = std::make_unique<RunningFleet>(m);
        uint32_t seg = 0;
        while (seg < n) {   // SEQUENTIAL runs optimistically, as in tree_select
            const uint32_t end = n;
            EventIndexView ixv;
            FleetView fv;
            sync_state(m, &ixv, &fv);
            sync_tenant_map(m);
            StringTreeView tv = tree.flush(lane.stream, &launches);
            StringSelectArgs a;
            a.text = lane.d_text.as<uint8_t>() - base; a.offsets = lane.d_offsets.as<uint32_t>();
            a.first = seg; a.count = end - seg;
            a.out_idx = lane.d_out.as<int32_t>(); a.out_info = lane.d_info.as<smgx_decision_info>();
            a.out_node = lane.d_path_len.as<uint32_t>(); a.out_tenant = lane.d_tenant.as<int32_t>(); a.out_fill = lane.d_fill.as<uint8_t>();
            a.cache_threshold = cfg.cache_threshold; a.decide = decide ? 1 : 0;
            launch_string_select(tv, fv, m.d_slice_of_tenant.as<int32_t>(), m.d_flags.as<uint8_t>(), (uint32_t)tenants.names.size(), a, lane.stream);
            ++launches;
            const uint32_t cnt = end - seg;
            SMGX_CUDA(cudaMemcpyAsync(out_idx + seg, lane.d_out.as<int32_t>() + seg, (size_t)cnt * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(info.data() + seg, lane.d_info.as<smgx_decision_info>() + seg, (size_t)cnt * sizeof(smgx_decision_info), cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(node.data() + seg, lane.d_path_len.as<uint32_t>() + seg, (size_t)cnt * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(ten.data() + seg, lane.d_tenant.as<int32_t>() + seg, (size_t)cnt * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(fill.data() + seg, lane.d_fill.as<uint8_t>() + seg, (size_t)cnt, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaStreamSynchronize(lane.stream));
            tree.begin_chunk();
            uint32_t r = seg;
            for (; r < end; ++r) {
                if (decide && info[r].branch == SMGX_BR_NO_HEALTHY) continue;
                int32_t pick = out_idx[r];
                uint8_t pick_br = info[r].branch;
                if (rf) decide_running(m, *rf, info[r].matched, info[r].input, ten[r], &pick, &pick_br);
                if (!snapshot && r > seg) {   // is the snapshot walk still the walk the reference would do now?
                    bool valid = true;
                    uint64_t sum_chars = 0;
                    for (uint32_t nd = node[r]; valid && nd != 0 && nd != kNoNode; nd = tree.parent_of(nd)) { valid = !tree.split_in_chunk(nd); sum_chars += tree.label_chars_of(nd); }
                    const uint8_t br = pick_br;
                    if (valid && (br == SMGX_BR_TREE_MATCH || br == SMGX_BR_TREE_FALLBACK_FIRST_HEALTHY)) valid = tree.any_tenant_of(node[r]) == ten[r];
                    if (valid && sum_chars == info[r].matched && info[r].matched < info[r].input) {   // stopped under a node: still no child for the next char?
                        const uint8_t* tx = text + offsets[r];
                        const uint32_t nb = offsets[r + 1] - offsets[r];
                        uint32_t pb = 0, chars = 0;
                        while (pb < nb && chars < info[r].matched) { ++pb; while (pb < nb && (tx[pb] & 0xC0) == 0x80) ++pb; ++chars; }
                        uint32_t cl;
                        if (pb < nb) valid = !tree.has_child(node[r], utf8_first(tx + pb, &cl));
                    }
                    if (!valid) break;
                }
                // cache fill, epoch draw, 1-in-8 refresh (:598-637): SNAPSHOT replays what the walk read, SEQUENTIAL what the node holds now
                if (snapshot) tree.apply_match_effects(node[r], ten[r], fill[r] != 0);
                else tree.apply_match_effects(node[r], tree.any_tenant_of(node[r]), !tree.cache_valid_of(node[r]));
                if (!decide) continue;
                if (rf) {
                    out_idx[r] = pick; info[r].branch = pick_br;
                    if (pick >= 0) rf->bump(pick);
                }
                const uint8_t br = info[r].branch;
                if ((br == SMGX_BR_TREE_MATCH || br == SMGX_BR_TREE_MIN_LOAD || br == SMGX_BR_IMBALANCED_MIN_LOAD) && out_idx[r] >= 0) {
                    const size_t idx = (size_t)out_idx[r];
                    const uint8_t* tx = text + offsets[r];
                    const uint32_t nb = offsets[r + 1] - offsets[r];
                    tree.insert_text(tx, nb, m.tenant_of_slice[idx]);   // :938 / :421
                    uint32_t pb = 0, chars = 0;   // text.chars().take(matched_char_count): byte length of the matched prefix
                    while (pb < nb && chars < info[r].matched) { ++pb; while (pb < nb && (tx[pb] & 0xC0) == 0x80) ++pb; ++chars; }
                    hash_index_put_text(m, path_hash[r], tx, pb);
                    if (idx < m.processed.size()) ++m.processed[idx];
                }
            }
            seg = r;
        }
        if (out_info) memcpy(out_info, info.data(), (size_t)n * sizeof(smgx_decision_info));
        if (out_tenant) memcpy(out_tenant, ten.data(), (size_t)n * 4);
    }

    // CacheAwarePolicy::evict_cache (cache_aware.rs:311-352); caller holds `mu`
    void evict_all(uint64_t max_size) {
        for (auto& kv : models) if (kv.second->string_tree) kv.second->string_tree->evict_tenant_by_size((size_t)max_size);   // :317-321
        for (auto& kv : models) if (kv.second->token_tree) kv.second->token_tree->evict_tenant_by_size((size_t)max_size);     // :322-326
        for (auto& kv : models) {   // per model, per tree kind (:335-351)
            if (kv.second->hash_index_text.size() > max_size) { kv.second->hash_index_text.clear(); kv.second->hash_arena_text.clear(); kv.second->hash_dead_text = 0; }
            if (kv.second->hash_index_tokens.size() > max_size) { kv.second->hash_index_tokens.clear(); kv.second->hash_arena_tokens.clear(); kv.second->hash_dead_tokens = 0; }
        }
    }
    // The reference's background eviction thread (cache_aware.rs:126-199): every eviction_interval_secs, bound every tree to
    // max_tree_size.  Host-side tree maintenance only — it issues no CUDA work; the mirrors pick the changes up at the next flush.
    void start_eviction_thread() {
        if (cfg.eviction_interval_secs == 0) return;
        evictor = std::thread([this]() {
            std::unique_lock<std::mutex> lk(evict_mu);
            while (!evict_stop) {
                if (evict_cv.wait_for(lk, std::chrono::seconds(cfg.eviction_interval_secs), [this] { return evict_stop; })) break;
                std::lock_guard<std::mutex> g(mu);
                evict_all(cfg.max_tree_size);
            }
        });
    }
    void stop_eviction_thread() {
        if (!evictor.joinable()) return;
        { std::lock_guard<std::mutex> lk(evict_mu); evict_stop = true; }
        evict_cv.notify_all();
        evictor.join();
    }

    Lane& free_lane() {
        for (auto& l : lanes) if (!l.busy) return l;
        throw Error(SMGX_BUSY, "all pipeline lanes are in flight; call smgx_wait first");
    }

    uint64_t submit_host(ModelState& m, const uint32_t* tokens, const uint32_t* offsets, uint32_t n, int32_t* out_idx, smgx_decision_info* out_info) {
        SMGX_REQUIRE(n <= cfg.max_batch, "batch larger than max_batch");
        // load feedback: the imbalance gate is re-evaluated per request by the in-order pass, so an event-mode model always takes the event path;
        // the tree update of the picks that did take the imbalanced branch is applied when the ticket is waited for
        const bool fb_event = load_feedback && has_event_indexer(m);
        if (!fb_event && (!has_event_indexer(m) || (host_imbalanced(m) && m.token_tree))) {
            // approximate token tree (or the imbalanced path's tree update): completes synchronously
            for (uint32_t i = 0; i < n; ++i) SMGX_REQUIRE(offsets[i + 1] >= offsets[i], "offsets must be non-decreasing");
            Lane& l = free_lane();   // SMGX_BUSY must be raised BEFORE the tree is touched: callers retry the whole batch on BUSY
            tree_select(m, tokens, offsets, n, out_idx, out_info, true, nullptr, nullptr, &l);   // on the lane just reserved: its staging is idle
            l.busy = true; l.ticket = ++ticket_seq; l.model = &m; l.host_out = out_idx; l.n = 0;   // n = 0: processed already counted
            return l.ticket;
        }
        SMGX_REQUIRE(m.urls.size() > 0 || true, "");
        Lane& lane = free_lane();
        uint32_t max_len = 0;
        for (uint32_t i = 0; i < n; ++i) {
            SMGX_REQUIRE(offsets[i + 1] >= offsets[i], "offsets must be non-decreasing");
            max_len = std::max(max_len, offsets[i + 1] - offsets[i]);
        }
        SMGX_REQUIRE(max_len <= cfg.max_tokens_per_request, "request longer than max_tokens_per_request");
        uint64_t total = n ? offsets[n] : 0;
        uint64_t base = n ? offsets[0] : 0;
        lane.d_tokens.reserve(std::max<uint64_t>(total - base, 1) * 4 + 16);
        lane.d_offsets.reserve(((size_t)n + 1) * 4);
        lane.d_out.reserve(std::max<uint32_t>(n, 1) * 4);
        smgx_decision_info* info_host = out_info;
        if (fb_event && !out_info && m.token_tree) { lane.fb_info.resize(std::max<uint32_t>(n, 1)); info_host = lane.fb_info.data(); }   // branches are needed at wait()
        if (info_host) lane.d_info.reserve(std::max<uint32_t>(n, 1) * sizeof(smgx_decision_info));
        if (n) {
            // tokens are copied from offsets[0]; the kernel indexes with the caller's absolute offsets
            SMGX_CUDA(cudaMemcpyAsync(lane.d_tokens.ptr, tokens + base, (total - base) * 4, cudaMemcpyHostToDevice, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(lane.d_offsets.ptr, offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, lane.stream));
            enqueue_tokens(m, lane, lane.d_tokens.as<uint32_t>() - base, lane.d_offsets.as<uint32_t>(), n, std::max<uint32_t>(max_len, 1),
                           lane.d_out.as<int32_t>(), info_host ? lane.d_info.as<smgx_decision_info>() : nullptr);
            SMGX_CUDA(cudaMemcpyAsync(out_idx, lane.d_out.ptr, (size_t)n * 4, cudaMemcpyDeviceToHost, lane.stream));
            if (info_host)
                SMGX_CUDA(cudaMemcpyAsync(info_host, lane.d_info.ptr, (size_t)n * sizeof(smgx_decision_info), cudaMemcpyDeviceToHost, lane.stream));
        }
        lane.busy = true;
        lane.ticket = ++ticket_seq;
        lane.model = &m;
        lane.host_out = out_idx;
        lane.n = n;
        lane.slice_version = m.slice_version;
        lane.fb_tokens = (fb_event && m.token_tree) ? tokens : nullptr;
        lane.fb_offsets = offsets;
        lane.fb_info_host = info_host;
        return lane.ticket;
    }

    void wait(uint64_t ticket) {
        for (auto& l : lanes) {
            if (!l.busy || l.ticket != ticket) continue;
            SMGX_CUDA(cudaStreamSynchronize(l.stream));
            l.busy = false;
            // increment_processed(): every event-mode / imbalanced pick increments (cache_aware.rs:437, :767, :829).  The picks index the
            // slice of the submission: after smgx_set_workers replaced it (and reset the counters) they name no worker of the new slice.
            ModelState& m = *l.model;
            const uint32_t credit = l.slice_version == m.slice_version ? l.n : 0;
            for (uint32_t i = 0; i < credit; ++i) {
                int32_t idx = l.host_out[i];
                if (idx >= 0 && (size_t)idx < m.processed.size()) ++m.processed[(size_t)idx];
            }
            if (l.fb_tokens && l.fb_info_host && m.token_tree) {
                // load-feedback batches: the picks that took the imbalanced branch still owe select_worker_min_load's tree update (cache_aware.rs:380-402)
                std::vector<uint32_t> toks, offs{0};
                std::vector<int32_t> forced;
                std::vector<uint32_t> who;
                for (uint32_t i = 0; i < l.n; ++i) {
                    if (l.fb_info_host[i].branch != SMGX_BR_IMBALANCED_MIN_LOAD || l.host_out[i] < 0) continue;
                    toks.insert(toks.end(), l.fb_tokens + l.fb_offsets[i], l.fb_tokens + l.fb_offsets[i + 1]);
                    offs.push_back((uint32_t)toks.size());
                    forced.push_back(l.host_out[i]);
                    who.push_back(i);
                }
                const ModelState* mp = &m;
                l.fb_tokens = nullptr;
                if (!forced.empty()) {
                    std::vector<int32_t> scratch(forced.size());
                    std::vector<smgx_decision_info> sub(forced.size());
                    smgx_decision_info* dst = l.fb_info_host;
                    uint32_t dummy = 0;
                    tree_select(const_cast<ModelState&>(*mp), toks.empty() ? &dummy : toks.data(), offs.data(), (uint32_t)forced.size(), scratch.data(), sub.data(), false, nullptr,
                                forced.data(), &l);
                    for (size_t k = 0; k < who.size(); ++k) { dst[who[k]].matched = sub[k].matched; dst[who[k]].nodes = sub[k].nodes; }   // select_worker_min_load reports the tree match (:380-395)
                }
            }
            return;
        }
        throw Error(SMGX_INVALID_ARGUMENT, "unknown or already completed ticket");
    }

    // Peer-memory exchange of the worker-id-sharded pick: every rank owns one symmetric gather buffer (two parities);
    // rank g's candidates are stored straight into slot g of every rank's buffer over NVLink (CUDA IPC mappings).
    struct Exchange {
        uint32_t world = 0, rank = 0, max_batch = 0;
        DevBuf local, d_bases, d_cand, d_fleet, d_arrive, d_gbase;
        std::vector<uint8_t*> peer;       // peer[q] = rank q's buffer as mapped here (own = local.ptr)
        std::vector<bool> opened;
        uint64_t seq = 0;
        size_t flag_off = 0, fleet_off = 0, cand_off = 0, parity_stride = 0, cand_slot_bytes = 0;
        static constexpr uint32_t kFleetStride = 64;
        bool connected = false;
    } xch;

    TenantTable tenants;         // TENANT_INTERN_POOL (token_tree.rs:160-176)
    uint64_t token_ts = 0;       // GLOBAL_TIMESTAMP (token_tree.rs:179), shared by every token tree of the policy
    uint64_t string_epoch = 0;   // EPOCH_COUNTER (string_tree.rs:239), shared by every string tree of the policy
    uint32_t tree_batch_mode = SMGX_TREE_BATCH_SEQUENTIAL;
    bool load_feedback = false;   // event-driven calls as a request stream (smgx_set_load_feedback, or the CACHE_AWARE bit)
    bool tree_feedback = false;   // token-tree / string-tree calls as a request stream (the CACHE_AWARE bit of smgx_set_load_feedback_policies)
    bool prefix_feedback = false; // prefix_hash calls as a request stream (SMGX_FEEDBACK_PREFIX_HASH)
    bool p2c_feedback = false;    // power_of_two calls as a request stream (SMGX_FEEDBACK_POWER_OF_TWO)
    uint32_t walk_chunk_seq = 0;
    smgx_cache_aware_config cfg;
    int sm_count = 132;              // H100 SXM; replaced by the device's own count when a device is opened
    size_t l2_bytes = 50u << 20;
    std::mutex mu;
    std::thread evictor;
    std::mutex evict_mu;
    std::condition_variable evict_cv;
    bool evict_stop = false;
    std::map<std::string, std::unique_ptr<ModelState>> models;
    bool monitor = false;
    std::vector<Lane> lanes;
    cudaStream_t ctrl = nullptr;
    cudaEvent_t state_ready = nullptr;
    DevBuf d_err, d_flush, scratch, scratch2, d_gbase, d_done_counters;
    static constexpr uint32_t kDoneCounters = 256;   // completion counters of mapped submissions in flight (one per launch, reused round-robin)
    uint64_t done_seq = 0, mapped_seq = 0;
    uint64_t launches = 0;
    uint64_t ticket_seq = 0;
};

}  // namespace smgx

// =================================================================================================================
// C ABI
// =================================================================================================================
using namespace smgx;

struct smgx_policy {
    Policy impl;
    explicit smgx_policy(const smgx_cache_aware_config& c) : impl(c) { impl.start_eviction_thread(); }
};

namespace {
void set_err(char** err, const std::string& msg) {
    if (!err) return;
    char* s = (char*)malloc(msg.size() + 1);
    if (s) memcpy(s, msg.c_str(), msg.size() + 1);
    *err = s;
}
template <class F> smgx_status guard(char** err, F&& f) {
    if (err) *err = nullptr;
    try {
        return f();
    } catch (const Error& e) {
        set_err(err, e.what());
        return e.code;
    } catch (const std::bad_alloc&) {
        set_err(err, "out of memory");
        return SMGX_MEMORY_ERROR;
    } catch (const std::exception& e) {
        set_err(err, e.what());
        return SMGX_UNKNOWN_ERROR;
    }
}
#define NONNULL(p) SMGX_REQUIRE((p) != nullptr, "Invalid arguments: null pointer")
}  // namespace

extern "C" {

void smgx_default_config(smgx_cache_aware_config* c) {
    if (!c) return;
    c->cache_threshold = 0.5f; c->balance_abs_threshold = 32; c->balance_rel_threshold = 1.1f;
    c->eviction_interval_secs = 30; c->max_tree_size = 10000; c->block_size = 16;
    c->device_id = 0; c->max_batch = 65536; c->max_tokens_per_request = 32768; c->tree_batch_mode = SMGX_TREE_BATCH_SEQUENTIAL;
}

smgx_policy* smgx_policy_create(const smgx_cache_aware_config* cfg, char** err) {
    smgx_policy* out = nullptr;
    guard(err, [&]() {
        NONNULL(cfg);
        out = new smgx_policy(*cfg);
        return SMGX_SUCCESS;
    });
    return out;
}
void smgx_policy_free(smgx_policy* p) { delete p; }
const char* smgx_policy_name(void) { return "cache_aware"; }
uint32_t smgx_abi_version(void) { return SMGX_ABI_VERSION; }
void smgx_free_string(char* s) { free(s); }
void* smgx_alloc_pinned(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
    return p;
}
void smgx_free_pinned(void* ptr) { if (ptr) cudaFreeHost(ptr); }

// Bind the CALLING thread (and, by first touch / preferred policy, the pinned buffers it allocates afterwards) to the NUMA node the
// device hangs off: a rank whose staging memory sits on the other socket pays for every H2D copy twice (UPI hop).  Opt-in, process-local.
smgx_status smgx_bind_numa(int device_id, int* out_node, char** err) {
    return guard(err, [&]() {
        if (out_node) *out_node = -1;
        char bus[32] = {0};
        SMGX_CUDA(cudaDeviceGetPCIBusId(bus, sizeof(bus), device_id));
        for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
        int node = -1;
        {
            std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
            FILE* f = fopen(path.c_str(), "r");
            if (f) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
        }
        if (node < 0) return SMGX_SUCCESS;   // single-node box or no topology information: nothing to do
        cpu_set_t set;
        CPU_ZERO(&set);
        int n_cpu = 0;
        {
            std::string path = "/sys/devices/system/node/node" + std::to_string(node) + "/cpulist";
            FILE* f = fopen(path.c_str(), "r");
            if (f) {
                int a, b;
                for (;;) {
                    if (fscanf(f, "%d", &a) != 1) break;
                    b = a;
                    int ch = fgetc(f);
                    if (ch == '-') { if (fscanf(f, "%d", &b) != 1) b = a; ch = fgetc(f); }
                    for (int c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET(c, &set); ++n_cpu; }
                    if (ch != ',') break;
                }
                fclose(f);
            }
        }
        if (n_cpu > 0) {
            cpu_set_t cur;   // intersect with what the process is allowed to use (containers)
            CPU_ZERO(&cur);
            if (sched_getaffinity(0, sizeof(cur), &cur) == 0) {
                cpu_set_t both;
                CPU_AND(&both, &cur, &set);
                if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof(both), &both);
            }
        }
        if (node < 64) {
            unsigned long mask = 1ul << node;
            syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, sizeof(mask) * 8);
        }
        if (out_node) *out_node = node;
        return SMGX_SUCCESS;
    });
}


// ---- fleet ----
smgx_status smgx_set_workers(smgx_policy* p, const char* model_key, const char* const* urls, uint32_t n, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || urls != nullptr, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        m.urls.clear();
        for (uint32_t i = 0; i < n; ++i) { NONNULL(urls[i]); m.urls.emplace_back(urls[i]); }
        m.loads.assign(n, 0);
        m.flags.assign(n, 3);
        m.processed.assign(n, 0);
        ++m.slice_version;
        m.fleet_dirty = true;
        m.fleet_dirty_tenant = true;
        m.pf_struct_dirty = m.pf_state_dirty = true;
        p->impl.tree_of(m, true);                                   // init_workers creates the trees (cache_aware.rs:231-247)
        StringTreeIndex& st = p->impl.stree_of(m);
        for (auto& u : m.urls) st.insert_text(nullptr, 0, p->impl.tenants.intern(u));   // tree.insert_text("", url) (:239, :275)
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_set_fleet_state(smgx_policy* p, const char* model_key, const uint64_t* loads, const uint8_t* healthy, const uint8_t* circuit_ok,
                                 uint32_t n, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        SMGX_REQUIRE(n == m.urls.size(), "fleet state length does not match the worker slice");
        for (uint32_t i = 0; i < n; ++i) {
            if (loads) m.loads[i] = loads[i];
            uint8_t h = healthy ? (healthy[i] ? 1 : 0) : (m.flags[i] & 1);
            uint8_t c = circuit_ok ? (circuit_ok[i] ? 2 : 0) : (m.flags[i] & 2);   // null = keep the previous circuit-breaker bit
            m.flags[i] = h | c;
        }
        m.fleet_dirty = true;
        m.pf_state_dirty = true;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_add_worker(smgx_policy* p, const char* model_key, const char* url, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(url);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        if (std::find(m.urls.begin(), m.urls.end(), url) == m.urls.end()) {
            m.urls.emplace_back(url); m.loads.push_back(0); m.flags.push_back(3); m.processed.push_back(0);
            m.fleet_dirty = true;
            m.fleet_dirty_tenant = true;
            m.pf_struct_dirty = m.pf_state_dirty = true;
        }
        p->impl.tree_of(m, true);
        p->impl.stree_of(m).insert_text(nullptr, 0, p->impl.tenants.intern(url));   // add_worker_by_url (:269-283)
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_remove_worker(smgx_policy* p, const char* model_key, const char* url, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(url);
        (void)model_key;  // no-op, as in the reference (cache_aware.rs:285-308): stale entries die by eviction
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_take_processed(smgx_policy* p, const char* model_key, uint64_t* out_counts, uint32_t n, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        for (uint32_t i = 0; i < n && i < m.processed.size(); ++i) { if (out_counts) out_counts[i] = m.processed[i]; m.processed[i] = 0; }
        return SMGX_SUCCESS;
    });
}

// ---- event index ----
smgx_status smgx_set_kv_event_monitor(smgx_policy* p, int present, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.monitor = present != 0;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_create(smgx_policy* p, const char* model_key, uint32_t jump_size, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        m.indexer = std::make_unique<EventIndex>(jump_size);
        m.indexer->device_enabled = p->impl.cfg.device_id >= 0;
        m.seen_workers_version = ~0ULL;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_set_block_size(smgx_policy* p, const char* model_key, uint32_t block_size, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        m.has_learned_bs = true;
        m.learned_bs = block_size;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_intern_worker(smgx_policy* p, const char* model_key, const char* url, uint32_t* out_id, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(url); NONNULL(out_id);
        std::lock_guard<std::mutex> g(p->impl.mu);
        *out_id = p->impl.indexer(model_key).intern_worker(url);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_worker_id(smgx_policy* p, const char* model_key, const char* url, int64_t* out_id, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(url); NONNULL(out_id);
        std::lock_guard<std::mutex> g(p->impl.mu);
        *out_id = p->impl.indexer(model_key).worker_id(url);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_apply_stored(smgx_policy* p, const char* model_key, uint32_t worker_id, const uint64_t* seq_hashes,
                                      const uint64_t* content_hashes, uint32_t n_blocks, const uint64_t* parent_seq_hash, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n_blocks == 0 || (seq_hashes && content_hashes), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        smgx_status st = p->impl.indexer(model_key).apply_stored(worker_id, seq_hashes, content_hashes, n_blocks, parent_seq_hash);
        if (st == SMGX_WORKER_NOT_TRACKED) set_err(err, "worker not tracked in index");          // event_tree.rs:100
        if (st == SMGX_PARENT_BLOCK_NOT_FOUND) set_err(err, "parent block hash not found for worker");  // :101
        return st;
    });
}
smgx_status smgx_indexer_apply_removed(smgx_policy* p, const char* model_key, uint32_t worker_id, const uint64_t* seq_hashes, uint32_t n, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || seq_hashes, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.indexer(model_key).apply_removed(worker_id, seq_hashes, n);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_apply_cleared(smgx_policy* p, const char* model_key, uint32_t worker_id, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.indexer(model_key).apply_cleared(worker_id);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_remove_worker(smgx_policy* p, const char* model_key, uint32_t worker_id, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.indexer(model_key).remove_worker(worker_id);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_current_size(smgx_policy* p, const char* model_key, uint64_t* out, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out);
        std::lock_guard<std::mutex> g(p->impl.mu);
        *out = p->impl.indexer(model_key).current_size();
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_indexer_entry_count(smgx_policy* p, const char* model_key, uint64_t* out, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out);
        std::lock_guard<std::mutex> g(p->impl.mu);
        *out = p->impl.indexer(model_key).entry_count();
        return SMGX_SUCCESS;
    });
}

smgx_status smgx_content_hashes(smgx_policy* p, const uint32_t* tokens, uint32_t n_tokens, uint32_t block_size, uint64_t* out_hashes,
                                uint32_t cap, uint32_t* out_n, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_n);
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        uint32_t nb = block_size ? n_tokens / block_size : 0;
        *out_n = nb;
        if (nb == 0) return SMGX_SUCCESS;
        NONNULL(tokens); NONNULL(out_hashes);
        SMGX_REQUIRE(cap >= nb, "output capacity too small");
        Lane& l = P.lanes[0];
        P.scratch.reserve((size_t)n_tokens * 4);
        P.scratch2.reserve((size_t)nb * 8);
        SMGX_CUDA(cudaMemcpyAsync(P.scratch.ptr, tokens, (size_t)n_tokens * 4, cudaMemcpyHostToDevice, l.stream));
        launch_content_hashes(P.scratch.as<uint32_t>(), n_tokens, block_size, P.scratch2.as<uint64_t>(), l.stream);
        ++P.launches;
        SMGX_CUDA(cudaMemcpyAsync(out_hashes, P.scratch2.ptr, (size_t)nb * 8, cudaMemcpyDeviceToHost, l.stream));
        SMGX_CUDA(cudaStreamSynchronize(l.stream));
        return SMGX_SUCCESS;
    });
}

smgx_status smgx_indexer_apply_stored_tokens(smgx_policy* p, const char* model_key, uint32_t worker_id, const uint64_t* seq_hashes,
                                             const uint32_t* token_ids, uint32_t block_size, uint32_t n_blocks, const uint64_t* parent_seq_hash,
                                             char** err) {
    // convert_kv_block hashes token_ids (kv_event_monitor.rs:592-597); done by the content-hash kernel, then apply_stored.
    if (err) *err = nullptr;
    if (!p) { set_err(err, "Invalid arguments: null pointer"); return SMGX_INVALID_ARGUMENT; }
    if (n_blocks == 0) return SMGX_SUCCESS;
    if (block_size == 0) { set_err(err, "block_size must be > 0"); return SMGX_INVALID_ARGUMENT; }
    std::vector<uint64_t> hashes(n_blocks);
    uint32_t got = 0;
    smgx_status st = smgx_content_hashes(p, token_ids, n_blocks * block_size, block_size, hashes.data(), n_blocks, &got, err);
    if (st != SMGX_SUCCESS) return st;
    return smgx_indexer_apply_stored(p, model_key, worker_id, seq_hashes, hashes.data(), n_blocks, parent_seq_hash, err);
}

// KvEventMonitor::apply_event for a batch of events of one model (worker/kv_event_monitor.rs:525-597): every stored block's
// token_ids are hashed in ONE kernel launch (convert_kv_block :592-597), then the events are applied in order on the
// host-authoritative index — Stored with the fresh-chain retry on WorkerNotTracked / ParentBlockNotFound (:559-571), Removed, Cleared.
smgx_status smgx_kv_events_apply(smgx_policy* p, const char* model_key, const smgx_kv_event* events, uint32_t n_events, const int64_t* block_hashes,
                                 const uint32_t* block_tok_offsets, const uint32_t* token_ids, uint32_t n_blocks, uint32_t* out_fallbacks, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n_events == 0 || events, "Invalid arguments: null pointer");
        SMGX_REQUIRE(n_blocks == 0 || (block_hashes && block_tok_offsets), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        EventIndex& ix = P.indexer(model_key);
        std::vector<uint64_t> content(n_blocks);
        uint32_t n_stored = 0;
        for (uint32_t e = 0; e < n_events; ++e) {
            SMGX_REQUIRE(events[e].kind <= SMGX_KV_CLEARED, "unknown event kind");
            if (events[e].kind != SMGX_KV_CLEARED) SMGX_REQUIRE((uint64_t)events[e].first_block + events[e].n_blocks <= n_blocks, "event block range out of bounds");
            if (events[e].kind == SMGX_KV_STORED) n_stored += events[e].n_blocks;
        }
        if (n_stored) {   // hash every block of the batch (removed events' slots are hashed too when they carry tokens; they are ignored below)
            P.use_device();
            for (uint32_t j = 0; j < n_blocks; ++j) SMGX_REQUIRE(block_tok_offsets[j + 1] >= block_tok_offsets[j], "block token offsets must be non-decreasing");
            const uint32_t n_tok = block_tok_offsets[n_blocks];
            SMGX_REQUIRE(n_tok == 0 || token_ids, "Invalid arguments: null pointer");
            Lane& l = P.lanes[0];
            P.scratch.reserve(std::max<size_t>((size_t)n_tok, 1) * 4 + ((size_t)n_blocks + 1) * 4 + 64);
            P.scratch2.reserve((size_t)n_blocks * 8);
            uint32_t* d_tok = P.scratch.as<uint32_t>();
            uint32_t* d_off = d_tok + std::max<uint32_t>(n_tok, 1);
            if (n_tok) SMGX_CUDA(cudaMemcpyAsync(d_tok, token_ids, (size_t)n_tok * 4, cudaMemcpyHostToDevice, l.stream));
            SMGX_CUDA(cudaMemcpyAsync(d_off, block_tok_offsets, ((size_t)n_blocks + 1) * 4, cudaMemcpyHostToDevice, l.stream));
            launch_content_hashes_ragged(d_tok, d_off, n_blocks, P.scratch2.as<uint64_t>(), l.stream);
            ++P.launches;
            SMGX_CUDA(cudaMemcpyAsync(content.data(), P.scratch2.ptr, (size_t)n_blocks * 8, cudaMemcpyDeviceToHost, l.stream));
            SMGX_CUDA(cudaStreamSynchronize(l.stream));
        }
        uint32_t fallbacks = 0;
        std::vector<uint64_t> seq;
        for (uint32_t e = 0; e < n_events; ++e) {
            const smgx_kv_event& ev = events[e];
            if (ev.kind == SMGX_KV_CLEARED) { ix.apply_cleared(ev.worker_id); continue; }
            seq.resize(ev.n_blocks);
            for (uint32_t j = 0; j < ev.n_blocks; ++j) seq[j] = (uint64_t)block_hashes[ev.first_block + j];   // SequenceHash::from(i64): bit reinterpretation (:643)
            if (ev.kind == SMGX_KV_REMOVED) { ix.apply_removed(ev.worker_id, seq.data(), ev.n_blocks); continue; }
            const uint64_t parent = (uint64_t)ev.parent_block_hash;
            smgx_status st = ix.apply_stored(ev.worker_id, seq.data(), content.data() + ev.first_block, ev.n_blocks, ev.has_parent ? &parent : nullptr);
            if (st == SMGX_WORKER_NOT_TRACKED || st == SMGX_PARENT_BLOCK_NOT_FOUND) {   // cold start or parent evicted: start a new chain
                ++fallbacks;
                ix.apply_stored(ev.worker_id, seq.data(), content.data() + ev.first_block, ev.n_blocks, nullptr);
            }
        }
        if (out_fallbacks) *out_fallbacks = fallbacks;
        return SMGX_SUCCESS;
    });
}

smgx_status smgx_indexer_find_matches(smgx_policy* p, const char* model_key, const uint64_t* content_hashes, uint32_t n, int early_exit,
                                      uint32_t* out_scores, uint64_t* out_tree_sizes, uint32_t cap, uint32_t* out_n_workers, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_scores); NONNULL(out_n_workers);
        SMGX_REQUIRE(n == 0 || content_hashes, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        if (!m.indexer) throw Error(SMGX_NOT_FOUND, "no event indexer for this model");
        uint32_t nw = m.indexer->n_workers();
        *out_n_workers = nw;
        SMGX_REQUIRE(cap >= nw, "output capacity smaller than the worker count");
        EventIndexView ixv;
        P.sync_state(m, &ixv, nullptr);
        Lane& l = P.lanes[0];
        size_t score_slots = (size_t)std::max<uint32_t>(ixv.words * 64, 64);
        P.scratch.reserve(std::max<size_t>((size_t)n, 1) * 8);
        P.scratch2.reserve(score_slots * 4);
        if (n) SMGX_CUDA(cudaMemcpyAsync(P.scratch.ptr, content_hashes, (size_t)n * 8, cudaMemcpyHostToDevice, l.stream));
        SMGX_CUDA(cudaMemsetAsync(P.scratch2.ptr, 0, score_slots * 4, l.stream));
        launch_find_matches(ixv, P.scratch.as<uint64_t>(), n, early_exit != 0, P.scratch2.as<uint32_t>(), l.stream);
        ++P.launches;
        std::vector<uint32_t> sc(score_slots);
        SMGX_CUDA(cudaMemcpyAsync(sc.data(), P.scratch2.ptr, score_slots * 4, cudaMemcpyDeviceToHost, l.stream));
        std::vector<uint64_t> ts(std::max<uint32_t>(nw, 1));
        if (nw) SMGX_CUDA(cudaMemcpyAsync(ts.data(), ixv.tree_sizes, (size_t)nw * 8, cudaMemcpyDeviceToHost, l.stream));
        SMGX_CUDA(cudaStreamSynchronize(l.stream));
        for (uint32_t w = 0; w < nw; ++w) { out_scores[w] = sc[w]; if (out_tree_sizes) out_tree_sizes[w] = ts[w]; }
        return SMGX_SUCCESS;
    });
}

// ---- approximate token tree: kv_index::TokenTree (crates/kv_index/src/token_tree.rs) ----
smgx_status smgx_tree_create(smgx_policy* p, const char* model_key, int eviction_policy, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(eviction_policy >= 0 && eviction_policy <= 5, "unknown eviction policy");
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        m.token_tree = std::make_unique<TokenTreeIndex>(&p->impl.tenants, &p->impl.token_ts, (EvictPolicy)eviction_policy);
        m.token_tree->device_enabled = p->impl.cfg.device_id >= 0;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tree_insert_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, uint32_t n, const char* tenant, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(tenant);
        SMGX_REQUIRE(n == 0 || tokens, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        TokenTreeIndex& t = p->impl.tree_of(m, true);
        if (n >= kPage) t.insert_tokens(tokens, n, p->impl.tenants.intern(tenant));   // shorter inputs return before interning (:403-410)
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tree_insert_tokens_batch(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint64_t* offsets, uint32_t n,
                                          const char* const* tenants, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (tokens && offsets && tenants), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        TokenTreeIndex& t = p->impl.tree_of(m, true);
        for (uint32_t i = 0; i < n; ++i) {
            NONNULL(tenants[i]);
            SMGX_REQUIRE(offsets[i + 1] >= offsets[i], "offsets must be non-decreasing");
            const uint64_t len = offsets[i + 1] - offsets[i];
            if (len >= kPage) t.insert_tokens(tokens + offsets[i], (size_t)len, p->impl.tenants.intern(tenants[i]));
        }
        return SMGX_SUCCESS;
    });
}
// Read-only walk + pick of device-resident batches against the current tree (no touches, no inserts): the K2a kernel by itself.
smgx_status smgx_tree_walk_many_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint32_t* const* d_tokens,
                                       const uint32_t* const* d_offsets, const uint32_t* n, int32_t* const* d_out_worker_idx,
                                       smgx_decision_info* const* d_out_info, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n_batches == 0 || (d_tokens && d_offsets && n && d_out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        TokenTreeIndex& tree = P.tree_of(m, false);
        EventIndexView ixv;
        FleetView fv;
        P.sync_state(m, &ixv, &fv);
        P.sync_tenant_map(m);
        if (tree.pending()) {   // mirror update in ctrl-stream order, then every lane waits for it
            for (auto& l : P.lanes) if (l.has_done) SMGX_CUDA(cudaStreamWaitEvent(P.ctrl, l.done, 0));
            tree.flush(P.ctrl, &P.launches);
            SMGX_CUDA(cudaEventRecord(P.state_ready, P.ctrl));
            for (auto& l : P.lanes) SMGX_CUDA(cudaStreamWaitEvent(l.stream, P.state_ready, 0));
        }
        const TokenTreeView tv = tree.flush(P.ctrl, &P.launches);   // nothing pending: returns the view
        for (uint32_t j = 0; j < n_batches; ++j) {   // one launch per batch, round-robin over the stream lanes
            Lane& lane = P.lanes[(P.walk_chunk_seq++) % P.lanes.size()];
            TreeSelectArgs a{};
            a.tokens = d_tokens[j]; a.offsets = d_offsets[j]; a.first = 0; a.count = n[j];
            a.out_idx = d_out_worker_idx[j]; a.out_info = d_out_info ? d_out_info[j] : nullptr;
            a.cache_threshold = P.cfg.cache_threshold; a.decide = 1;
            launch_tree_select(tv, fv, m.d_slice_of_tenant.as<int32_t>(), m.d_flags.as<uint8_t>(), (uint32_t)P.tenants.names.size(), a, lane.stream);
            ++P.launches;
            SMGX_CUDA(cudaEventRecord(lane.done, lane.stream));
            lane.has_done = true;
        }
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tree_match_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, uint32_t n, uint32_t* out_matched,
                                   uint32_t* out_input, char* out_tenant, uint32_t tenant_cap, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_matched); NONNULL(out_input);
        SMGX_REQUIRE(n == 0 || tokens, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, true);
        P.tree_of(m, true);
        uint32_t offs[2] = {0, n};
        uint32_t dummy = 0;
        int32_t idx = -1, ten = -1;
        smgx_decision_info di{};
        P.tree_select(m, n ? tokens : &dummy, offs, 1, &idx, &di, false, &ten);
        *out_matched = di.matched;
        *out_input = di.input;
        if (out_tenant && tenant_cap) {
            std::string name = "empty";
            if (ten >= 0) name = P.tenants.names[(size_t)ten];
            else if (n < kPage) { int32_t rt = m.token_tree->any_tenant(0); if (rt >= 0) name = P.tenants.names[(size_t)rt]; }   // :620-629
            size_t k = std::min<size_t>(name.size(), tenant_cap - 1);
            memcpy(out_tenant, name.data(), k);
            out_tenant[k] = 0;
        }
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tree_evict_tenant(smgx_policy* p, const char* model_key, const char* tenant, uint64_t max_tokens, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(tenant);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        int64_t t = p->impl.tenants.find(tenant);
        if (t >= 0 && m.token_tree) m.token_tree->evict_tenant((uint32_t)t, (size_t)max_tokens);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_evict_cache(smgx_policy* p, uint64_t max_size, char** err) {   // CacheAwarePolicy::evict_cache (cache_aware.rs:311-352)
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.evict_all(max_size);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tree_tenant_size(smgx_policy* p, const char* model_key, const char* tenant, uint64_t* out, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(tenant); NONNULL(out);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        int64_t t = p->impl.tenants.find(tenant);
        *out = (t >= 0 && m.token_tree) ? m.token_tree->tenant_token_size((uint32_t)t) : 0;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tree_clear(smgx_policy* p, const char* model_key, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        if (m.token_tree) m.token_tree->clear();
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tree_entries(smgx_policy* p, const char* model_key, char** out_text, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_text);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        std::string s;
        if (m.token_tree) {
            std::vector<std::pair<std::vector<uint32_t>, std::vector<std::pair<uint32_t, uint64_t>>>> es;
            m.token_tree->entries(es);
            for (auto& e : es) {
                for (size_t i = 0; i < e.first.size(); ++i) { if (i) s.push_back(','); s += std::to_string(e.first[i]); }
                s.push_back('|');
                for (size_t i = 0; i < e.second.size(); ++i) { if (i) s.push_back(';'); s += p->impl.tenants.names[e.second[i].first] + "=" + std::to_string(e.second[i].second); }
                s.push_back('\n');
            }
        }
        char* c = (char*)malloc(s.size() + 1);
        if (!c) throw std::bad_alloc();
        memcpy(c, s.c_str(), s.size() + 1);
        *out_text = c;
        return SMGX_SUCCESS;
    });
}

// ---- tokenizer ----
static std::vector<std::pair<std::string, uint32_t>> collect_specials(const char* const* strs, const uint32_t* ids, uint32_t n) {
    std::vector<std::pair<std::string, uint32_t>> sp;
    SMGX_REQUIRE(n == 0 || (strs && ids), "Invalid arguments: null pointer");
    for (uint32_t i = 0; i < n; ++i) { SMGX_REQUIRE(strs[i] != nullptr, "Invalid arguments: null pointer"); sp.emplace_back(strs[i], ids[i]); }
    return sp;
}
// smgx_pretokenizer → Pretok; an unknown value is an invalid argument
static Pretok pretok_of(smgx_pretokenizer pt) {
    SMGX_REQUIRE(pt == SMGX_PRETOK_CL100K || pt == SMGX_PRETOK_R50K || pt == SMGX_PRETOK_QWEN2 || pt == SMGX_PRETOK_DEEPSEEK,
                 "Invalid arguments: unknown pretokenizer " + std::to_string((int)pt));
    return pt == SMGX_PRETOK_R50K ? Pretok::R50k : pt == SMGX_PRETOK_QWEN2 ? Pretok::Qwen2 : pt == SMGX_PRETOK_DEEPSEEK ? Pretok::DeepSeek : Pretok::Cl100k;
}
smgx_status smgx_tokenizer_load_tiktoken_file_ex(smgx_policy* p, const char* model_key, const char* path, const char* const* special_strs,
                                                 const uint32_t* special_ids, uint32_t n_special, smgx_pretokenizer pretokenizer, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(path);
        const Pretok pt = pretok_of(pretokenizer);
        std::lock_guard<std::mutex> g(p->impl.mu);
        bool dev = p->impl.cfg.device_id >= 0;
        if (dev) p->impl.use_device();
        ModelState& m = p->impl.model(model_key, true);
        m.tokenizer.reset(Tokenizer::from_tiktoken_file(path, collect_specials(special_strs, special_ids, n_special), dev, pt));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tokenizer_load_tiktoken_file(smgx_policy* p, const char* model_key, const char* path, const char* const* special_strs,
                                              const uint32_t* special_ids, uint32_t n_special, char** err) {
    return smgx_tokenizer_load_tiktoken_file_ex(p, model_key, path, special_strs, special_ids, n_special, SMGX_PRETOK_CL100K, err);
}
smgx_status smgx_tokenizer_load_tiktoken_ex(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets,
                                            const uint32_t* ranks, uint32_t n_tokens, const char* const* special_strs,
                                            const uint32_t* special_ids, uint32_t n_special, smgx_pretokenizer pretokenizer, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(blob); NONNULL(tok_offsets); NONNULL(ranks);
        const Pretok pt = pretok_of(pretokenizer);
        std::lock_guard<std::mutex> g(p->impl.mu);
        bool dev = p->impl.cfg.device_id >= 0;
        if (dev) p->impl.use_device();
        std::vector<std::string> toks(n_tokens);
        std::vector<uint32_t> rk(ranks, ranks + n_tokens);
        for (uint32_t i = 0; i < n_tokens; ++i) toks[i].assign((const char*)blob + tok_offsets[i], tok_offsets[i + 1] - tok_offsets[i]);
        ModelState& m = p->impl.model(model_key, true);
        m.tokenizer.reset(new Tokenizer(toks, rk, collect_specials(special_strs, special_ids, n_special), dev, pt));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tokenizer_load_tiktoken(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets,
                                         const uint32_t* ranks, uint32_t n_tokens, const char* const* special_strs,
                                         const uint32_t* special_ids, uint32_t n_special, char** err) {
    return smgx_tokenizer_load_tiktoken_ex(p, model_key, blob, tok_offsets, ranks, n_tokens, special_strs, special_ids, n_special, SMGX_PRETOK_CL100K, err);
}

smgx_status smgx_tokenizer_load_bpe_merges(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                           uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, int ignore_merges, const char* const* special_strs,
                                           const uint32_t* special_ids, uint32_t n_special, char** err) {
    return smgx_tokenizer_load_bpe_merges_ex(p, model_key, blob, tok_offsets, ids, n_tokens, merges, n_merges, ignore_merges, special_strs, special_ids,
                                             n_special, SMGX_PRETOK_CL100K, err);
}
smgx_status smgx_tokenizer_load_bpe_merges_ex(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                              uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, int ignore_merges, const char* const* special_strs,
                                              const uint32_t* special_ids, uint32_t n_special, smgx_pretokenizer pretokenizer, char** err) {
    return smgx_tokenizer_load_bpe_merges_norm(p, model_key, blob, tok_offsets, ids, n_tokens, merges, n_merges, ignore_merges, special_strs, special_ids,
                                               n_special, pretokenizer, SMGX_NORMALIZER_NONE, err);
}
smgx_status smgx_tokenizer_load_bpe_merges_norm(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                                uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, int ignore_merges, const char* const* special_strs,
                                                const uint32_t* special_ids, uint32_t n_special, smgx_pretokenizer pretokenizer, smgx_normalizer normalizer,
                                                char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(blob); NONNULL(tok_offsets); NONNULL(ids);
        SMGX_REQUIRE(n_merges == 0 || merges, "Invalid arguments: null pointer");
        const Pretok pt = pretok_of(pretokenizer);
        SMGX_REQUIRE(normalizer == SMGX_NORMALIZER_NONE || normalizer == SMGX_NORMALIZER_NFC, "Invalid arguments: unknown normalizer " + std::to_string((int)normalizer));
        std::lock_guard<std::mutex> g(p->impl.mu);
        bool dev = p->impl.cfg.device_id >= 0;
        if (dev) p->impl.use_device();
        std::vector<std::string> toks(n_tokens);
        std::vector<uint32_t> id(ids, ids + n_tokens);
        for (uint32_t i = 0; i < n_tokens; ++i) toks[i].assign((const char*)blob + tok_offsets[i], tok_offsets[i + 1] - tok_offsets[i]);
        std::vector<std::pair<uint32_t, uint32_t>> mg(n_merges);
        for (uint32_t i = 0; i < n_merges; ++i) mg[i] = {merges[2 * i], merges[2 * i + 1]};
        ModelState& m = p->impl.model(model_key, true);
        m.tokenizer.reset(new Tokenizer(toks, id, mg, ignore_merges != 0, collect_specials(special_strs, special_ids, n_special), dev, pt,
                                        normalizer == SMGX_NORMALIZER_NFC));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_tokenizer_load_bpe_metaspace(smgx_policy* p, const char* model_key, const uint8_t* blob, const uint32_t* tok_offsets, const uint32_t* ids,
                                              uint32_t n_tokens, const uint32_t* merges, uint32_t n_merges, const char* const* special_strs,
                                              const uint32_t* special_ids, uint32_t n_special, smgx_sp_shape shape, smgx_prepend_scheme prepend_scheme,
                                              int split, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(blob); NONNULL(tok_offsets); NONNULL(ids);
        SMGX_REQUIRE(n_merges == 0 || merges, "Invalid arguments: null pointer");
        SMGX_REQUIRE(shape == SMGX_SP_LEGACY || shape == SMGX_SP_METASPACE, "Invalid arguments: unknown shape " + std::to_string((int)shape));
        SMGX_REQUIRE(prepend_scheme == SMGX_PREPEND_NEVER || prepend_scheme == SMGX_PREPEND_FIRST || prepend_scheme == SMGX_PREPEND_ALWAYS,
                     "Invalid arguments: unknown prepend_scheme " + std::to_string((int)prepend_scheme));
        SMGX_REQUIRE(split == 0 || split == 1, "Invalid arguments: split must be 0 or 1, not " + std::to_string(split));
        SMGX_REQUIRE(shape == SMGX_SP_METASPACE || (prepend_scheme == SMGX_PREPEND_ALWAYS && split == 0),
                     "Invalid arguments: the legacy shape takes prepend_scheme SMGX_PREPEND_ALWAYS and split 0");
        MetaspaceMode ms{1, shape == SMGX_SP_LEGACY ? (uint32_t)MS_PREPEND_LEGACY
                            : prepend_scheme == SMGX_PREPEND_NEVER ? (uint32_t)MS_PREPEND_NEVER
                            : prepend_scheme == SMGX_PREPEND_FIRST ? (uint32_t)MS_PREPEND_FIRST : (uint32_t)MS_PREPEND_ALWAYS,
                         (uint32_t)split};
        std::lock_guard<std::mutex> g(p->impl.mu);
        bool dev = p->impl.cfg.device_id >= 0;
        if (dev) p->impl.use_device();
        std::vector<std::string> toks(n_tokens);
        std::vector<uint32_t> id(ids, ids + n_tokens);
        for (uint32_t i = 0; i < n_tokens; ++i) toks[i].assign((const char*)blob + tok_offsets[i], tok_offsets[i + 1] - tok_offsets[i]);
        std::vector<std::pair<uint32_t, uint32_t>> mg(n_merges);
        for (uint32_t i = 0; i < n_merges; ++i) mg[i] = {merges[2 * i], merges[2 * i + 1]};
        ModelState& m = p->impl.model(model_key, true);
        m.tokenizer.reset(new Tokenizer(toks, id, mg, collect_specials(special_strs, special_ids, n_special), dev, ms));
        return SMGX_SUCCESS;
    });
}

// H2D the ragged text and tokenise it on `lane`; returns the device token buffers (valid until the lane is reused).
static void tokenize_on_lane(Policy& P, ModelState& m, Lane& lane, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                             uint32_t* max_text_len) {
    if (!m.tokenizer) throw Error(SMGX_NOT_FOUND, "no tokenizer loaded for this model");
    uint32_t mx = 0;
    for (uint32_t i = 0; i < n; ++i) {
        SMGX_REQUIRE(offsets[i + 1] >= offsets[i], "offsets must be non-decreasing");
        mx = std::max(mx, offsets[i + 1] - offsets[i]);
    }
    *max_text_len = mx;
    const uint32_t base = n ? offsets[0] : 0, total = n ? offsets[n] - base : 0;
    lane.d_text.reserve(std::max<uint32_t>(total, 1) + 16);
    lane.d_offsets.reserve(((size_t)n + 1) * 4);
    lane.d_toff.reserve(((size_t)n + 1) * 4);
    lane.d_tokens.reserve((size_t)std::max<uint32_t>(total, 1) * m.tokenizer->growth() * 4 + 16);   // growth(): most tokens per byte
    if (n == 0) return;
    if (total) SMGX_CUDA(cudaMemcpyAsync(lane.d_text.ptr, text + base, total, cudaMemcpyHostToDevice, lane.stream));
    SMGX_CUDA(cudaMemcpyAsync(lane.d_offsets.ptr, offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, lane.stream));
    // kernels index text with the caller's absolute offsets
    m.tokenizer->encode_batch(lane.d_text.as<uint8_t>() - base, lane.d_offsets.as<uint32_t>(), n, base, total + base, mx, lane.d_tokens.as<uint32_t>(),
                              lane.d_toff.as<uint32_t>(), lane.tok_scratch, lane.stream, &P.launches);
}

// Token bound of the text-in pick for requests of at most mx bytes: mx without a normalizer (a byte is at most one token); with one,
// growth() × mx capped at max_tokens_per_request — a request longer than that after normalization takes the device-side over-length
// treatment (pick -1, branch 255, error flag) instead of a write past its hash row.
static uint32_t text_token_bound(const Policy& P, const ModelState& m, uint32_t mx) {
    const uint64_t b = (uint64_t)mx * m.tokenizer->growth();
    return std::max<uint32_t>((uint32_t)std::min<uint64_t>(b, std::max<uint64_t>(mx, P.cfg.max_tokens_per_request)), 1);
}
static bool text_may_exceed(const Policy& P, const ModelState& m, uint32_t mx) { return (uint64_t)mx * m.tokenizer->growth() > P.cfg.max_tokens_per_request; }

static void copy_tokens_out(Lane& lane, uint32_t n, uint32_t* out_tokens, uint32_t* out_tok_offsets, uint32_t cap_tokens) {
    std::vector<uint32_t> toff_local;
    uint32_t* toff = out_tok_offsets;
    if (!toff) { toff_local.resize((size_t)n + 1); toff = toff_local.data(); }
    SMGX_CUDA(cudaMemcpyAsync(toff, lane.d_toff.ptr, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, lane.stream));
    SMGX_CUDA(cudaStreamSynchronize(lane.stream));
    if (out_tokens) {
        SMGX_REQUIRE(toff[n] <= cap_tokens, "out_tokens capacity too small");
        if (toff[n]) SMGX_CUDA(cudaMemcpyAsync(out_tokens, lane.d_tokens.ptr, (size_t)toff[n] * 4, cudaMemcpyDeviceToHost, lane.stream));
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
    }
}

smgx_status smgx_tokenize_batch(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                uint32_t* out_tokens, uint32_t* out_tok_offsets, uint32_t cap_tokens, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_tok_offsets);
        SMGX_REQUIRE(n == 0 || (text && offsets && out_tokens), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        Lane& lane = P.free_lane();
        uint32_t mx = 0;
        if (n == 0) { out_tok_offsets[0] = 0; return SMGX_SUCCESS; }
        tokenize_on_lane(P, m, lane, text, offsets, n, &mx);
        copy_tokens_out(lane, n, out_tokens, out_tok_offsets, cap_tokens);
        return SMGX_SUCCESS;
    });
}

static smgx_status select_batch_text_once(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                          int32_t* out_worker_idx, smgx_decision_info* out_info, uint32_t* out_tokens, uint32_t* out_tok_offsets,
                                          uint32_t cap_tokens, char** err);
smgx_status smgx_select_batch_text(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                   int32_t* out_worker_idx, smgx_decision_info* out_info, uint32_t* out_tokens, uint32_t* out_tok_offsets,
                                   uint32_t cap_tokens, char** err) {
    for (;;) {   // synchronous: wait for a lane when other threads hold them all
        const smgx_status st = select_batch_text_once(p, model_key, text, offsets, n, out_worker_idx, out_info, out_tokens, out_tok_offsets, cap_tokens, err);
        if (st != SMGX_BUSY) return st;
        if (err && *err) { smgx_free_string(*err); *err = nullptr; }
        std::this_thread::yield();
    }
}
static smgx_status select_batch_text_once(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                          int32_t* out_worker_idx, smgx_decision_info* out_info, uint32_t* out_tokens, uint32_t* out_tok_offsets,
                                          uint32_t cap_tokens, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (text && offsets && out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(n <= P.cfg.max_batch, "batch larger than max_batch");
        ModelState& m = P.model(model_key, false);
        if (n == 0) { if (out_tok_offsets) out_tok_offsets[0] = 0; return SMGX_SUCCESS; }
        Lane& lane = P.free_lane();
        uint32_t mx = 0;
        tokenize_on_lane(P, m, lane, text, offsets, n, &mx);
        SMGX_REQUIRE(mx <= P.cfg.max_tokens_per_request, "request longer than max_tokens_per_request");
        if (!P.has_event_indexer(m) || (P.host_imbalanced(m) && m.token_tree)) {
            // approximate token tree on the tokens just produced: the host-side updater needs them, so they come back first
            std::vector<uint32_t> toff(n + 1);
            SMGX_CUDA(cudaMemcpyAsync(toff.data(), lane.d_toff.ptr, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaStreamSynchronize(lane.stream));
            std::vector<uint32_t> toks(std::max<uint32_t>(toff[n], 1));
            if (toff[n]) SMGX_CUDA(cudaMemcpy(toks.data(), lane.d_tokens.ptr, (size_t)toff[n] * 4, cudaMemcpyDeviceToHost));
            if (out_tok_offsets) memcpy(out_tok_offsets, toff.data(), ((size_t)n + 1) * 4);
            if (out_tokens) { SMGX_REQUIRE(toff[n] <= cap_tokens, "token output buffer too small"); memcpy(out_tokens, toks.data(), (size_t)toff[n] * 4); }
            if (P.tree_feedback && P.has_event_indexer(m)) P.wait(P.submit_host(m, toks.data(), toff.data(), n, out_worker_idx, out_info));   // the gate is per request: the event-driven stream
            else P.tree_select(m, toks.data(), toff.data(), n, out_worker_idx, out_info, true, nullptr);
            return SMGX_SUCCESS;
        }
        lane.d_out.reserve((size_t)n * 4);
        if (out_info) lane.d_info.reserve((size_t)n * sizeof(smgx_decision_info));
        // a request of b bytes has at most growth() × b tokens → bounds the per-request hash row
        const bool may_overflow = text_may_exceed(P, m, mx);
        P.enqueue_tokens(m, lane, lane.d_tokens.as<uint32_t>(), lane.d_toff.as<uint32_t>(), n, text_token_bound(P, m, mx), lane.d_out.as<int32_t>(),
                         out_info ? lane.d_info.as<smgx_decision_info>() : nullptr);
        SMGX_CUDA(cudaMemcpyAsync(out_worker_idx, lane.d_out.ptr, (size_t)n * 4, cudaMemcpyDeviceToHost, lane.stream));
        if (out_info)
            SMGX_CUDA(cudaMemcpyAsync(out_info, lane.d_info.ptr, (size_t)n * sizeof(smgx_decision_info), cudaMemcpyDeviceToHost, lane.stream));
        if (out_tokens || out_tok_offsets) copy_tokens_out(lane, n, out_tokens, out_tok_offsets, cap_tokens);
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
        for (uint32_t i = 0; i < n; ++i) {
            int32_t idx = out_worker_idx[i];
            if (idx >= 0 && (size_t)idx < m.processed.size()) ++m.processed[(size_t)idx];
        }
        if (may_overflow) {   // a request over max_tokens_per_request only after normalization: reported by this call, once
            uint32_t flag = 0;
            SMGX_CUDA(cudaMemcpy(&flag, P.d_err.ptr, 4, cudaMemcpyDeviceToHost));
            if (flag & kErrNoSlowKernel) {
                SMGX_CUDA(cudaMemset(P.d_err.ptr, 0, 4));
                throw Error(SMGX_UNKNOWN_ERROR, "internal error: a request needed event_slow_kernel in a launch that did not run it");
            }
            if (flag == 1) {
                SMGX_CUDA(cudaMemset(P.d_err.ptr, 0, 4));
                throw Error(SMGX_INVALID_ARGUMENT, "a request exceeded max_tokens_per_request after normalization");
            }
        }
        return SMGX_SUCCESS;
    });
}

// ---- string tree: kv_index::Tree (crates/kv_index/src/string_tree.rs) ----
static char* dup_cstr(const std::string& s) {
    char* c = (char*)malloc(s.size() + 1);
    if (!c) throw std::bad_alloc();
    memcpy(c, s.data(), s.size());
    c[s.size()] = 0;
    return c;
}
smgx_status smgx_stree_insert_text(smgx_policy* p, const char* model_key, const uint8_t* text, uint32_t n_bytes, const char* tenant, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(tenant);
        SMGX_REQUIRE(n_bytes == 0 || text, "Invalid arguments: null pointer");
        SMGX_REQUIRE(StringTreeIndex::valid_utf8(text, n_bytes), "text is not valid UTF-8");
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        p->impl.stree_of(m).insert_text(text, n_bytes, p->impl.tenants.intern(tenant));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_stree_match(smgx_policy* p, const char* model_key, const uint8_t* text, uint32_t n_bytes, uint32_t* out_matched_chars,
                             uint32_t* out_input_chars, char* out_tenant, uint32_t tenant_cap, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_matched_chars); NONNULL(out_input_chars);
        SMGX_REQUIRE(n_bytes == 0 || text, "Invalid arguments: null pointer");
        SMGX_REQUIRE(StringTreeIndex::valid_utf8(text, n_bytes), "text is not valid UTF-8");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, true);
        uint32_t offs[2] = {0, n_bytes};
        uint8_t dummy = 0;
        int32_t idx = -1, ten = -1;
        smgx_decision_info di{};
        P.text_select(m, n_bytes ? text : &dummy, offs, 1, &idx, &di, false, &ten);
        *out_matched_chars = di.matched;
        *out_input_chars = di.input;
        if (out_tenant && tenant_cap) {
            const std::string name = ten >= 0 ? P.tenants.names[(size_t)ten] : std::string("empty");
            const size_t k = std::min<size_t>(name.size(), tenant_cap - 1);
            memcpy(out_tenant, name.data(), k);
            out_tenant[k] = 0;
        }
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_stree_prefix_match_tenant(smgx_policy* p, const char* model_key, const uint8_t* text, uint32_t n_bytes, const char* tenant,
                                           uint32_t* out_matched_bytes, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(tenant); NONNULL(out_matched_bytes);
        SMGX_REQUIRE(n_bytes == 0 || text, "Invalid arguments: null pointer");
        SMGX_REQUIRE(StringTreeIndex::valid_utf8(text, n_bytes), "text is not valid UTF-8");
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        uint8_t dummy = 0;
        *out_matched_bytes = (uint32_t)p->impl.stree_of(m).prefix_match_tenant(n_bytes ? text : &dummy, n_bytes, p->impl.tenants.find(tenant)).size();
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_stree_sizes(smgx_policy* p, const char* model_key, int maintained, char** out_text, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_text);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        StringTreeIndex& t = p->impl.stree_of(m);
        std::string s;
        for (auto& kv : (maintained ? t.tenant_char_counts() : t.used_size_per_tenant())) s += kv.first + "=" + std::to_string(kv.second) + "\n";
        *out_text = dup_cstr(s);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_stree_entries(smgx_policy* p, const char* model_key, char** out_text, uint64_t* out_len, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_text); NONNULL(out_len);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        std::vector<std::pair<std::string, std::vector<std::pair<uint32_t, uint64_t>>>> es;
        p->impl.stree_of(m).entries(es);
        std::string s;
        for (auto& e : es) {
            s += e.first; s.push_back('\x1f');
            for (size_t i = 0; i < e.second.size(); ++i) { if (i) s.push_back(';'); s += p->impl.tenants.names[e.second[i].first] + "=" + std::to_string(e.second[i].second); }
            s.push_back('\x1e');
        }
        *out_text = dup_cstr(s);
        *out_len = s.size();
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_stree_snapshot(smgx_policy* p, const char* model_key, char** out_bytes, uint64_t* out_len, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_bytes); NONNULL(out_len);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        std::string b;
        p->impl.stree_of(m).snapshot_bytes(b);
        *out_bytes = dup_cstr(b);
        *out_len = b.size();
        return SMGX_SUCCESS;
    });
}
static smgx_status stree_apply_snapshot(smgx_policy* p, const char* model_key, const uint8_t* bytes, uint64_t n, bool merge, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || bytes, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        StringTreeIndex& t = p->impl.stree_of(m);
        const bool ok = merge ? t.merge_snapshot(bytes, n) : t.load_snapshot(bytes, n);
        if (!ok) throw Error(SMGX_INVALID_ARGUMENT, "malformed TreeSnapshot (bincode)");
        m.fleet_dirty_tenant = true;   // new tenants may have been interned
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_stree_load_snapshot(smgx_policy* p, const char* model_key, const uint8_t* bytes, uint64_t n_bytes, char** err) {
    return stree_apply_snapshot(p, model_key, bytes, n_bytes, false, err);
}
smgx_status smgx_stree_merge_snapshot(smgx_policy* p, const char* model_key, const uint8_t* bytes, uint64_t n_bytes, char** err) {
    return stree_apply_snapshot(p, model_key, bytes, n_bytes, true, err);
}
smgx_status smgx_stree_clear(smgx_policy* p, const char* model_key, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        if (m.string_tree) m.string_tree->clear();
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_stree_node_count(smgx_policy* p, const char* model_key, uint64_t* out, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        *out = m.string_tree ? m.string_tree->node_count() : 0;
        return SMGX_SUCCESS;
    });
}

// ---- mesh path hashes + hash_index (crates/mesh/src/hash.rs:22-52; cache_aware.rs:95-101) ----
static smgx_status hash_paths(smgx_policy* p, const uint8_t* data, const uint32_t* offsets, uint32_t n, uint32_t elem_bytes, uint64_t* out, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (offsets && out), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        if (n == 0) return SMGX_SUCCESS;
        for (uint32_t i = 0; i < n; ++i) SMGX_REQUIRE(offsets[i + 1] >= offsets[i], "offsets must be non-decreasing");
        Lane& lane = P.lanes[0];
        const uint64_t base = (uint64_t)offsets[0] * elem_bytes, total = (uint64_t)(offsets[n] - offsets[0]) * elem_bytes;
        SMGX_REQUIRE(total == 0 || data, "Invalid arguments: null pointer");
        lane.d_text.reserve(std::max<uint64_t>(total, 1) + 16);
        lane.d_offsets.reserve(((size_t)n + 1) * 4);
        if (total) SMGX_CUDA(cudaMemcpyAsync(lane.d_text.ptr, data + base, total, cudaMemcpyHostToDevice, lane.stream));
        SMGX_CUDA(cudaMemcpyAsync(lane.d_offsets.ptr, offsets, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, lane.stream));
        std::vector<uint64_t> h;
        P.enqueue_path_hashes(lane, lane.d_text.as<uint8_t>() - base, lane.d_offsets.as<uint32_t>(), offsets, n, elem_bytes, h);
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
        memcpy(out, h.data(), (size_t)n * 8);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_hash_token_paths(smgx_policy* p, const uint32_t* tokens, const uint32_t* offsets, uint32_t n, uint64_t* out_hashes, char** err) {
    return hash_paths(p, reinterpret_cast<const uint8_t*>(tokens), offsets, n, 4, out_hashes, err);
}
smgx_status smgx_hash_node_paths(smgx_policy* p, const uint8_t* text, const uint32_t* offsets, uint32_t n, uint64_t* out_hashes, char** err) {
    return hash_paths(p, text, offsets, n, 1, out_hashes, err);
}
// ---- TreeHandle (cache_aware.rs:454-645): the mesh adapter's view of the policy ----
// apply_known_remote_insert (:499-551): resolve `node_hash` through hash_index[model] to the stored matched prefix and insert it for
// `worker_url`; false when the model, the hash or the tree is unknown (the caller then asks a peer for repair).
smgx_status smgx_tree_apply_known_remote_insert(smgx_policy* p, const char* model_key, int tree_kind, uint64_t node_hash, const char* worker_url,
                                                int* out_known, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(worker_url); NONNULL(out_known);
        SMGX_REQUIRE(tree_kind == 0 || tree_kind == 1, "tree_kind: 0 = String, 1 = Token");
        *out_known = 0;
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        auto it = P.models.find(norm_model(model_key));
        if (it == P.models.end()) return SMGX_SUCCESS;
        ModelState& m = *it->second;
        if (tree_kind == 0) {
            auto e = m.hash_index_text.find(node_hash);
            if (e == m.hash_index_text.end() || !m.string_tree) return SMGX_SUCCESS;
            const std::string path(m.hash_arena_text.data() + e->second.first, e->second.second);   // copy: the insert may not alias the arena
            m.string_tree->insert_text(reinterpret_cast<const uint8_t*>(path.data()), (uint32_t)path.size(), P.tenants.intern(worker_url));
        } else {
            auto e = m.hash_index_tokens.find(node_hash);
            if (e == m.hash_index_tokens.end() || !m.token_tree) return SMGX_SUCCESS;
            const std::vector<uint32_t> toks(m.hash_arena_tokens.begin() + (ptrdiff_t)e->second.first,
                                             m.hash_arena_tokens.begin() + (ptrdiff_t)(e->second.first + e->second.second));
            if (toks.size() >= kPage) m.token_tree->insert_tokens(toks.data(), toks.size(), P.tenants.intern(worker_url));   // shorter inputs return before interning (:403-410)
        }
        *out_known = 1;
        return SMGX_SUCCESS;
    });
}
// apply_repair_page (:575-645): every entry of the page's kind is inserted for each of its tenants (the tree is created on first use —
// repair is the cold-start path of a fresh peer) and its path hash (blake3 of the whole path, hashed on the GPU in one launch) is seeded
// into hash_index; entries of the other kind are skipped.  *out_applied = entries applied.
smgx_status smgx_tree_apply_repair_page(smgx_policy* p, const char* model_key, int tree_kind, const smgx_repair_entry* entries, uint32_t n,
                                        uint32_t* out_applied, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_applied);
        SMGX_REQUIRE(tree_kind == 0 || tree_kind == 1, "tree_kind: 0 = String, 1 = Token");
        SMGX_REQUIRE(n == 0 || entries, "Invalid arguments: null pointer");
        *out_applied = 0;
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        ModelState& m = P.model(model_key, true);
        if (tree_kind == 0) P.stree_of(m); else P.tree_of(m, true);
        // gather the page's entries of the right kind into one ragged buffer and hash their paths in one launch
        const uint32_t eb = tree_kind == 0 ? 1 : 4;
        std::vector<uint32_t> which;
        std::vector<uint32_t> offs{0};
        std::string blob;
        for (uint32_t i = 0; i < n; ++i) {
            if ((int)entries[i].kind != tree_kind) continue;   // variant mismatch: logged and skipped in the reference (:606-613, :633-640)
            SMGX_REQUIRE(entries[i].len == 0 || entries[i].data, "Invalid arguments: null pointer");
            SMGX_REQUIRE(entries[i].n_tenants == 0 || entries[i].tenants, "Invalid arguments: null pointer");
            which.push_back(i);
            blob.append(reinterpret_cast<const char*>(entries[i].data), (size_t)entries[i].len * eb);
            SMGX_REQUIRE(blob.size() / eb < (1ull << 32), "repair page too large");
            offs.push_back((uint32_t)(blob.size() / eb));
        }
        if (which.empty()) return SMGX_SUCCESS;
        P.use_device();
        std::vector<uint64_t> hashes;
        {
            Lane& lane = P.lanes[0];
            lane.d_text.reserve(std::max<size_t>(blob.size(), 1) + 16);
            lane.d_offsets.reserve(offs.size() * 4);
            if (!blob.empty()) SMGX_CUDA(cudaMemcpyAsync(lane.d_text.ptr, blob.data(), blob.size(), cudaMemcpyHostToDevice, lane.stream));
            SMGX_CUDA(cudaMemcpyAsync(lane.d_offsets.ptr, offs.data(), offs.size() * 4, cudaMemcpyHostToDevice, lane.stream));
            P.enqueue_path_hashes(lane, lane.d_text.as<uint8_t>(), lane.d_offsets.as<uint32_t>(), offs.data(), (uint32_t)which.size(), eb, hashes);
            SMGX_CUDA(cudaStreamSynchronize(lane.stream));
        }
        for (size_t k = 0; k < which.size(); ++k) {
            const smgx_repair_entry& e = entries[which[k]];
            for (uint32_t t = 0; t < e.n_tenants; ++t) {
                NONNULL(e.tenants[t]);
                if (tree_kind == 0) m.string_tree->insert_text(reinterpret_cast<const uint8_t*>(e.data), e.len, P.tenants.intern(e.tenants[t]));
                else if (e.len >= kPage) m.token_tree->insert_tokens(reinterpret_cast<const uint32_t*>(e.data), e.len, P.tenants.intern(e.tenants[t]));
            }
            if (tree_kind == 0) Policy::hash_index_put_text(m, hashes[k], reinterpret_cast<const uint8_t*>(e.data), e.len);
            else Policy::hash_index_put_tokens(m, hashes[k], reinterpret_cast<const uint32_t*>(e.data), e.len);
            ++*out_applied;
        }
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_hash_index_size(smgx_policy* p, const char* model_key, int text_kind, uint64_t* out, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        *out = text_kind ? m.hash_index_text.size() : m.hash_index_tokens.size();
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_hash_index_get(smgx_policy* p, const char* model_key, int text_kind, uint64_t path_hash, void* out, uint32_t cap_bytes,
                                uint32_t* out_bytes, int* out_found, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_bytes); NONNULL(out_found);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        *out_found = 0; *out_bytes = 0;
        const void* src = nullptr;
        size_t nb = 0;
        if (text_kind) { auto it = m.hash_index_text.find(path_hash); if (it != m.hash_index_text.end()) { src = m.hash_arena_text.data() + it->second.first; nb = it->second.second; *out_found = 1; } }
        else { auto it = m.hash_index_tokens.find(path_hash); if (it != m.hash_index_tokens.end()) { src = m.hash_arena_tokens.data() + it->second.first; nb = (size_t)it->second.second * 4; *out_found = 1; } }
        *out_bytes = (uint32_t)nb;
        if (*out_found && out && nb <= cap_bytes && nb) memcpy(out, src, nb);
        return SMGX_SUCCESS;
    });
}

// ---- adjacent policy: prefix_hash (model_gateway/src/policies/prefix_hash.rs) over the consistent hash ring (worker/hash_ring.rs) ----
smgx_status smgx_prefix_hash_configure(smgx_policy* p, uint64_t prefix_token_count, double load_factor, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(load_factor == load_factor, "load_factor is NaN");
        SMGX_REQUIRE(prefix_token_count <= 0xFFFFFFFFull, "prefix_token_count out of range");
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.prefix_token_count = prefix_token_count;
        p->impl.prefix_load_factor = load_factor;
        for (auto& kv : p->impl.models) kv.second->pf_state_dirty = true;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_hash_ring_set(smgx_policy* p, const char* model_key, const char* const* urls, uint32_t n, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || urls != nullptr, "Invalid arguments: null pointer");
        for (uint32_t i = 0; i < n; ++i) NONNULL(urls[i]);
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        P.ring_set(P.model(model_key, true), urls, n);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_hash_ring_clear(smgx_policy* p, const char* model_key, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, true);
        m.has_ring = false; m.ring_urls.clear(); m.ring_pos.clear(); m.ring_url.clear();
        m.pf_struct_dirty = true;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_hash_ring_entries(smgx_policy* p, const char* model_key, uint64_t* out_pos, uint32_t* out_url, uint32_t cap, uint32_t* out_len, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_len);
        std::lock_guard<std::mutex> g(p->impl.mu);
        ModelState& m = p->impl.model(model_key, false);
        if (!m.has_ring) throw Error(SMGX_NOT_FOUND, "no hash ring for this model");
        *out_len = (uint32_t)m.ring_pos.size();
        for (uint32_t i = 0; i < m.ring_pos.size() && i < cap; ++i) { if (out_pos) out_pos[i] = m.ring_pos[i]; if (out_url) out_url[i] = m.ring_url[i]; }
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_hash_ring_find_healthy(smgx_policy* p, const char* model_key, const uint8_t* keys, const uint32_t* key_offsets, uint32_t n,
                                        const uint8_t* url_ok, int32_t* out_url, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (key_offsets && out_url), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        if (!m.has_ring) throw Error(SMGX_NOT_FOUND, "no hash ring for this model");
        SMGX_REQUIRE(m.ring_urls.empty() || url_ok, "Invalid arguments: null pointer");
        if (n == 0) return SMGX_SUCCESS;
        for (uint32_t i = 0; i < n; ++i) SMGX_REQUIRE(key_offsets[i + 1] >= key_offsets[i], "offsets must be non-decreasing");
        SMGX_REQUIRE(key_offsets[n] == key_offsets[0] || keys, "Invalid arguments: null pointer");
        std::string blob(reinterpret_cast<const char*>(keys) + key_offsets[0], key_offsets[n] - key_offsets[0]);
        std::vector<uint32_t> offs(n + 1);
        for (uint32_t i = 0; i <= n; ++i) offs[i] = key_offsets[i] - key_offsets[0];
        std::vector<uint64_t> kp;
        P.ring_positions(blob, offs, kp);
        RingView rv; PrefixFleetView fv;
        P.sync_prefix(m, &rv, &fv);
        Lane& lane = P.lanes[0];
        const uint32_t nu = (uint32_t)m.ring_urls.size();
        P.scratch.reserve((size_t)n * 8 + std::max<uint32_t>(nu, 1) + 16);
        P.scratch2.reserve((size_t)n * 4);
        uint64_t* d_kp = P.scratch.as<uint64_t>();
        uint8_t* d_ok = reinterpret_cast<uint8_t*>(d_kp + n);
        SMGX_CUDA(cudaMemcpyAsync(d_kp, kp.data(), (size_t)n * 8, cudaMemcpyHostToDevice, lane.stream));
        if (nu) SMGX_CUDA(cudaMemcpyAsync(d_ok, url_ok, nu, cudaMemcpyHostToDevice, lane.stream));
        launch_ring_find(rv.pos, m.d_ring_url.as<uint32_t>(), rv.len, d_kp, d_ok, n, P.scratch2.as<int32_t>(), lane.stream);
        ++P.launches;
        SMGX_CUDA(cudaMemcpyAsync(out_url, P.scratch2.ptr, (size_t)n * 4, cudaMemcpyDeviceToHost, lane.stream));
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
        return SMGX_SUCCESS;
    });
}

// host-buffer forms: only the hashed prefix of each request is staged (pinned) and copied
static smgx_status prefix_host_call(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n, const uint8_t* has_tokens,
                                    int32_t* out_idx, smgx_decision_info* out_info, uint64_t* out_hash, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || offsets, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        if (n == 0) return SMGX_SUCCESS;
        SMGX_REQUIRE(n <= P.cfg.max_batch, "batch larger than max_batch");
        const uint32_t k = (uint32_t)P.prefix_token_count, keep = std::max(k, 1u);   // ≥ 1 token kept so that "tokens is empty" survives the packing
        uint64_t total = 0;
        for (uint32_t i = 0; i < n; ++i) { SMGX_REQUIRE(offsets[i + 1] >= offsets[i], "offsets must be non-decreasing"); total += std::min(offsets[i + 1] - offsets[i], keep); }
        SMGX_REQUIRE(total == 0 || tokens, "Invalid arguments: null pointer");
        const size_t off_bytes = ((size_t)n + 1) * 4, flag_bytes = has_tokens ? (((size_t)n + 3) & ~(size_t)3) : 0;
        P.pf_stage.reserve(total * 4 + off_bytes + flag_bytes + 16);
        uint32_t* h_tok = P.pf_stage.as<uint32_t>();
        uint32_t* h_off = h_tok + total;
        uint8_t* h_flag = reinterpret_cast<uint8_t*>(h_off + n + 1);
        uint64_t at = 0;
        for (uint32_t i = 0; i < n; ++i) {
            const uint32_t use = std::min(offsets[i + 1] - offsets[i], keep);
            h_off[i] = (uint32_t)at;
            if (use) memcpy(h_tok + at, tokens + offsets[i], (size_t)use * 4);
            at += use;
        }
        h_off[n] = (uint32_t)at;
        if (has_tokens) memcpy(h_flag, has_tokens, n);
        ModelState* m = out_idx ? &P.model(model_key, false) : nullptr;
        Lane& lane = P.lanes[0];
        const size_t in_bytes = total * 4 + off_bytes + flag_bytes;
        lane.d_tokens.reserve(in_bytes + 16);
        lane.d_out.reserve((size_t)n * 4);
        lane.d_info.reserve((size_t)n * sizeof(smgx_decision_info));
        lane.d_hashes.reserve((size_t)n * 8);
        SMGX_CUDA(cudaMemcpyAsync(lane.d_tokens.ptr, P.pf_stage.ptr, in_bytes, cudaMemcpyHostToDevice, lane.stream));
        RingView rv{nullptr, nullptr, 0, 0, nullptr, 63};
        PrefixFleetView fv{nullptr, nullptr, nullptr, nullptr, 0};
        if (m) P.sync_prefix(*m, &rv, &fv);
        PrefixArgs a;
        a.count = 1; a.prefix_tokens = k;
        uint32_t* d_tok = lane.d_tokens.as<uint32_t>();
        a.b[0].tokens = d_tok; a.b[0].offsets = d_tok + total;
        a.b[0].has_tokens = has_tokens ? reinterpret_cast<const uint8_t*>(d_tok + total + n + 1) : nullptr;
        a.b[0].out_idx = out_idx ? lane.d_out.as<int32_t>() : nullptr;
        a.b[0].out_info = out_info ? lane.d_info.as<smgx_decision_info>() : nullptr;
        a.b[0].hash = lane.d_hashes.as<uint64_t>();
        a.b[0].n = n;
        const bool fb = P.prefix_feedback && out_idx;
        if (fb) SMGX_REQUIRE(fv.n_slice <= kMaxFeedbackSlice, "fleet too large for the load-feedback pass");
        const PrefixFeedback pfb{P.prefix_load_factor, nullptr, 0};
        P.launches += launch_prefix_select(rv, fv, a, lane.stream, lane.stream, nullptr, fb ? &pfb : nullptr);
        const size_t hash_at = ((size_t)n * (4 + sizeof(smgx_decision_info)) + 7) & ~(size_t)7;
        P.pf_out.reserve(hash_at + (size_t)n * 8);
        int32_t* h_idx = P.pf_out.as<int32_t>();
        smgx_decision_info* h_info = reinterpret_cast<smgx_decision_info*>(h_idx + n);
        uint64_t* h_hash = reinterpret_cast<uint64_t*>(P.pf_out.as<uint8_t>() + hash_at);
        if (out_idx) SMGX_CUDA(cudaMemcpyAsync(h_idx, lane.d_out.ptr, (size_t)n * 4, cudaMemcpyDeviceToHost, lane.stream));
        if (out_info) SMGX_CUDA(cudaMemcpyAsync(h_info, lane.d_info.ptr, (size_t)n * sizeof(smgx_decision_info), cudaMemcpyDeviceToHost, lane.stream));
        if (out_hash) SMGX_CUDA(cudaMemcpyAsync(h_hash, lane.d_hashes.ptr, (size_t)n * 8, cudaMemcpyDeviceToHost, lane.stream));
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
        if (out_idx) memcpy(out_idx, h_idx, (size_t)n * 4);
        if (out_info) {
            memcpy(out_info, h_info, (size_t)n * sizeof(smgx_decision_info));
            for (uint32_t i = 0; i < n; ++i) out_info[i].input = offsets[i + 1] - offsets[i];   // the kernel saw the packed prefix only
        }
        if (out_hash) memcpy(out_hash, h_hash, (size_t)n * 8);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_prefix_hashes(smgx_policy* p, const uint32_t* tokens, const uint32_t* offsets, uint32_t n, uint64_t* out_hashes, char** err) {
    if (n && !out_hashes) { if (err) *err = dup_cstr("Invalid arguments: null pointer"); return SMGX_INVALID_ARGUMENT; }
    return prefix_host_call(p, "", tokens, offsets, n, nullptr, nullptr, nullptr, out_hashes, err);
}
smgx_status smgx_prefix_hash_select_batch_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n,
                                                 const uint8_t* has_tokens, int32_t* out_worker_idx, smgx_decision_info* out_info, char** err) {
    if (n && !out_worker_idx) { if (err) *err = dup_cstr("Invalid arguments: null pointer"); return SMGX_INVALID_ARGUMENT; }
    return prefix_host_call(p, model_key, tokens, offsets, n, has_tokens, out_worker_idx, out_info, nullptr, err);
}
smgx_status smgx_prefix_hash_select_many_tokens_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint32_t* const* d_tokens,
                                                       const uint32_t* const* d_offsets, const uint32_t* n, int32_t* const* d_out_worker_idx, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n_batches == 0 || (d_tokens && d_offsets && n && d_out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        RingView rv; PrefixFleetView fv;
        P.sync_prefix(m, &rv, &fv);
        // Groups of ≤ 32 batches: hash kernel on lane 0, pick kernel on lane 1 behind an event, so that the pick of group g runs beside
        // the hash kernel of group g + 1.  The hashes travel through two alternating scratch buffers; a buffer is reused only after
        // the pick that read it has finished (event wait on lane 0).
        Lane& lane = P.lanes[0];
        Lane& side = P.lanes.size() > 1 ? P.lanes[1] : P.lanes[0];
        // load feedback: every group's pick kernels run on `side` in order, each continuing from the running loads the previous one left
        const bool fb = P.prefix_feedback;
        if (fb) {
            SMGX_REQUIRE(fv.n_slice <= kMaxFeedbackSlice, "fleet too large for the load-feedback pass");
            if ((size_t)std::max<uint32_t>(fv.n_slice, 1) * 8 > P.pf_run_loads.cap) { SMGX_CUDA(cudaDeviceSynchronize()); P.pf_run_loads.reserve((size_t)std::max<uint32_t>(fv.n_slice, 1) * 8); }
        }
        for (uint32_t j0 = 0; j0 < n_batches; j0 += kMaxPrefixBatches) {
            PrefixArgs a;
            a.count = std::min<uint32_t>(kMaxPrefixBatches, n_batches - j0);
            a.prefix_tokens = (uint32_t)P.prefix_token_count;
            uint64_t total = 0;
            for (uint32_t k = 0; k < a.count; ++k) total += n[j0 + k];
            const uint32_t b = (uint32_t)(P.pf_group++ & 1);
            if (!P.pf_hash_ev[b]) { SMGX_CUDA(cudaEventCreateWithFlags(&P.pf_hash_ev[b], cudaEventDisableTiming)); SMGX_CUDA(cudaEventCreateWithFlags(&P.pf_pick_ev[b], cudaEventDisableTiming)); }
            if (P.pf_pick_pending[b]) SMGX_CUDA(cudaStreamWaitEvent(lane.stream, P.pf_pick_ev[b], 0));
            if (total * 8 > P.pf_hash_buf[b].cap) { SMGX_CUDA(cudaDeviceSynchronize()); P.pf_hash_buf[b].reserve(total * 8); }
            uint64_t at = 0;
            for (uint32_t k = 0; k < a.count; ++k) {
                a.b[k] = PrefixBatch{d_tokens[j0 + k], d_offsets[j0 + k], nullptr, d_out_worker_idx[j0 + k], nullptr, P.pf_hash_buf[b].as<uint64_t>() + at, n[j0 + k]};
                at += n[j0 + k];
            }
            const PrefixFeedback pfb{P.prefix_load_factor, P.pf_run_loads.as<uint64_t>(), j0 > 0 ? 1u : 0u};
            P.launches += launch_prefix_select(rv, fv, a, lane.stream, side.stream, P.pf_hash_ev[b], fb ? &pfb : nullptr);
            if (&side != &lane) { SMGX_CUDA(cudaEventRecord(P.pf_pick_ev[b], side.stream)); P.pf_pick_pending[b] = true; }
        }
        return SMGX_SUCCESS;
    });
}

// Read-only walk + pick of device-resident text batches against the current string tree: the K2c kernel by itself (bench).
smgx_status smgx_stree_walk_many_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint8_t* const* d_text,
                                        const uint32_t* const* d_offsets, const uint32_t* n, int32_t* const* d_out_worker_idx,
                                        smgx_decision_info* const* d_out_info, uint32_t* const* d_out_node, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n_batches == 0 || (d_text && d_offsets && n && d_out_worker_idx && d_out_node), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        StringTreeIndex& tree = P.stree_of(m);
        EventIndexView ixv;
        FleetView fv;
        P.sync_state(m, &ixv, &fv);
        P.sync_tenant_map(m);
        for (auto& l : P.lanes) if (l.has_done) SMGX_CUDA(cudaStreamWaitEvent(P.ctrl, l.done, 0));
        const StringTreeView tv = tree.flush(P.ctrl, &P.launches);
        SMGX_CUDA(cudaEventRecord(P.state_ready, P.ctrl));
        for (auto& l : P.lanes) SMGX_CUDA(cudaStreamWaitEvent(l.stream, P.state_ready, 0));
        for (uint32_t j = 0; j < n_batches; ++j) {
            Lane& lane = P.lanes[(P.walk_chunk_seq++) % P.lanes.size()];
            lane.d_tenant.reserve((size_t)std::max<uint32_t>(n[j], 1) * 4);
            lane.d_fill.reserve(std::max<uint32_t>(n[j], 1));
            StringSelectArgs a{};
            a.text = d_text[j]; a.offsets = d_offsets[j]; a.first = 0; a.count = n[j];
            a.out_idx = d_out_worker_idx[j]; a.out_info = d_out_info ? d_out_info[j] : nullptr;
            a.out_node = d_out_node[j]; a.out_tenant = lane.d_tenant.as<int32_t>(); a.out_fill = lane.d_fill.as<uint8_t>();
            a.cache_threshold = P.cfg.cache_threshold; a.decide = 1;
            launch_string_select(tv, fv, m.d_slice_of_tenant.as<int32_t>(), m.d_flags.as<uint8_t>(), (uint32_t)P.tenants.names.size(), a, lane.stream);
            ++P.launches;
            SMGX_CUDA(cudaEventRecord(lane.done, lane.stream));
            lane.has_done = true;
        }
        return SMGX_SUCCESS;
    });
}

smgx_status smgx_set_tree_batch_mode(smgx_policy* p, uint32_t mode, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(mode == SMGX_TREE_BATCH_SEQUENTIAL || mode == SMGX_TREE_BATCH_SNAPSHOT, "unknown tree batch mode");
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.tree_batch_mode = mode;
        return SMGX_SUCCESS;
    });
}

// select_worker with info.request_text = Some(text), info.tokens = None (HTTP routers): string tree (cache_aware.rs:688-689, :907-974)
smgx_status smgx_select_batch_request_text(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                                           int32_t* out_worker_idx, smgx_decision_info* out_info, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (text && offsets && out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(n <= P.cfg.max_batch, "batch larger than max_batch");
        ModelState& m = P.model(model_key, false);
        for (uint32_t i = 0; i < n; ++i) {
            SMGX_REQUIRE(offsets[i + 1] >= offsets[i], "offsets must be non-decreasing");
            SMGX_REQUIRE(StringTreeIndex::valid_utf8(text + offsets[i], offsets[i + 1] - offsets[i]), "request text is not valid UTF-8");
        }
        P.text_select(m, text, offsets, n, out_worker_idx, out_info, true, nullptr);
        return SMGX_SUCCESS;
    });
}

// Pipelined text-in pick: H2D of the text, tokenize, hash, search and the D2H of the picks are enqueued on one lane and the call
// returns; smgx_wait(ticket) completes it.  Event-driven mode only runs asynchronously — the tree modes need the tokens on the host
// for their updater and complete inside the call (the ticket is then already done).
smgx_status smgx_submit_text(smgx_policy* p, const char* model_key, const uint8_t* text, const uint32_t* offsets, uint32_t n,
                             int32_t* out_worker_idx, smgx_decision_info* out_info, uint64_t* out_ticket, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_ticket);
        SMGX_REQUIRE(n == 0 || (text && offsets && out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(n <= P.cfg.max_batch, "batch larger than max_batch");
        ModelState& m = P.model(model_key, false);
        Lane& lane = P.free_lane();
        uint32_t mx = 0;
        if (n) tokenize_on_lane(P, m, lane, text, offsets, n, &mx);
        SMGX_REQUIRE(mx <= P.cfg.max_tokens_per_request, "request longer than max_tokens_per_request");
        if (n && (!P.has_event_indexer(m) || (P.host_imbalanced(m) && m.token_tree))) {
            std::vector<uint32_t> toff(n + 1);
            SMGX_CUDA(cudaMemcpyAsync(toff.data(), lane.d_toff.ptr, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, lane.stream));
            SMGX_CUDA(cudaStreamSynchronize(lane.stream));
            std::vector<uint32_t> toks(std::max<uint32_t>(toff[n], 1));
            if (toff[n]) SMGX_CUDA(cudaMemcpy(toks.data(), lane.d_tokens.ptr, (size_t)toff[n] * 4, cudaMemcpyDeviceToHost));
            if (P.tree_feedback && P.has_event_indexer(m)) P.wait(P.submit_host(m, toks.data(), toff.data(), n, out_worker_idx, out_info));   // as in smgx_select_batch_text
            else P.tree_select(m, toks.data(), toff.data(), n, out_worker_idx, out_info, true, nullptr);
            Lane& l2 = P.free_lane();
            l2.busy = true; l2.ticket = ++P.ticket_seq; l2.model = &m; l2.host_out = out_worker_idx; l2.n = 0;   // processed already counted
            *out_ticket = l2.ticket;
            return SMGX_SUCCESS;
        }
        if (n) {
            lane.d_out.reserve((size_t)n * 4);
            if (out_info) lane.d_info.reserve((size_t)n * sizeof(smgx_decision_info));
            P.enqueue_tokens(m, lane, lane.d_tokens.as<uint32_t>(), lane.d_toff.as<uint32_t>(), n, text_token_bound(P, m, mx), lane.d_out.as<int32_t>(),
                             out_info ? lane.d_info.as<smgx_decision_info>() : nullptr);
            SMGX_CUDA(cudaMemcpyAsync(out_worker_idx, lane.d_out.ptr, (size_t)n * 4, cudaMemcpyDeviceToHost, lane.stream));
            if (out_info)
                SMGX_CUDA(cudaMemcpyAsync(out_info, lane.d_info.ptr, (size_t)n * sizeof(smgx_decision_info), cudaMemcpyDeviceToHost, lane.stream));
        }
        lane.busy = true;
        lane.ticket = ++P.ticket_seq;
        lane.model = &m;
        lane.host_out = out_worker_idx;
        lane.n = n;
        lane.slice_version = m.slice_version;
        *out_ticket = lane.ticket;
        return SMGX_SUCCESS;
    });
}

// ---- hot call ----
uint32_t smgx_pipeline_depth(const smgx_policy* p) { return p ? (uint32_t)p->impl.lanes.size() : 0; }

smgx_status smgx_submit_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n,
                               int32_t* out_worker_idx, smgx_decision_info* out_info, uint64_t* out_ticket, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_ticket);
        SMGX_REQUIRE(n == 0 || (tokens && offsets && out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.use_device();
        ModelState& m = p->impl.model(model_key, false);
        *out_ticket = p->impl.submit_host(m, tokens, offsets, n, out_worker_idx, out_info);
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_wait(smgx_policy* p, uint64_t ticket, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        // the stream is synchronised WITHOUT the policy mutex, so other threads keep submitting while this one waits
        cudaStream_t stream = nullptr;
        {
            std::lock_guard<std::mutex> g(p->impl.mu);
            p->impl.use_device();
            for (auto& l : p->impl.lanes) if (l.busy && l.ticket == ticket) stream = l.stream;
        }
        if (stream) SMGX_CUDA(cudaStreamSynchronize(stream));
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.wait(ticket);   // finds the lane again; its stream is idle now
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_set_load_feedback(smgx_policy* p, int enabled, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        std::lock_guard<std::mutex> g(p->impl.mu);
        p->impl.load_feedback = enabled != 0;
        p->impl.tree_feedback = p->impl.prefix_feedback = p->impl.p2c_feedback = false;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_set_load_feedback_policies(smgx_policy* p, uint32_t mask, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE((mask & ~(SMGX_FEEDBACK_CACHE_AWARE | SMGX_FEEDBACK_PREFIX_HASH | SMGX_FEEDBACK_POWER_OF_TWO)) == 0, "unknown load-feedback policy bit");
        std::lock_guard<std::mutex> g(p->impl.mu);
        const bool ca = (mask & SMGX_FEEDBACK_CACHE_AWARE) != 0;
        SMGX_REQUIRE(!(ca && p->impl.tree_batch_mode == SMGX_TREE_BATCH_SNAPSHOT),
                     "cache_aware load feedback does not combine with SMGX_TREE_BATCH_SNAPSHOT (use SEQUENTIAL)");
        p->impl.load_feedback = ca;
        p->impl.tree_feedback = ca;
        p->impl.prefix_feedback = (mask & SMGX_FEEDBACK_PREFIX_HASH) != 0;
        p->impl.p2c_feedback = (mask & SMGX_FEEDBACK_POWER_OF_TWO) != 0;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_select_batch_tokens(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n,
                                     int32_t* out_worker_idx, smgx_decision_info* out_info, char** err) {
    uint64_t t = 0;
    smgx_status st;
    for (;;) {   // a synchronous call simply waits for a lane when other threads hold them all
        st = smgx_submit_tokens(p, model_key, tokens, offsets, n, out_worker_idx, out_info, &t, err);
        if (st != SMGX_BUSY) break;
        if (err && *err) { smgx_free_string(*err); *err = nullptr; }
        std::this_thread::yield();
    }
    if (st != SMGX_SUCCESS) return st;
    return smgx_wait(p, t, err);
}

// Zero-copy submission for small, latency-bound batches: the kernel reads the caller's PINNED host buffers in place over PCIe, stores the
// picks straight back into pinned host memory and raises *done_flag = done_value when the whole batch is out — no staging copy, no
// cudaStreamSynchronize, no ticket.  Event-driven mode only (tree modes mutate host state: use smgx_submit_tokens).
smgx_status smgx_submit_tokens_mapped(smgx_policy* p, const char* model_key, const uint32_t* tokens, const uint32_t* offsets, uint32_t n,
                                      uint32_t max_request_tokens, int32_t* out_worker_idx, smgx_decision_info* out_info, uint64_t* done_flag,
                                      uint64_t done_value, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(done_flag);
        SMGX_REQUIRE(n == 0 || (tokens && offsets && out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        if (!P.has_event_indexer(m) || (P.host_imbalanced(m) && m.token_tree))
            throw Error(SMGX_NOT_FOUND, "mapped submissions serve the event-driven mode only; this model is routed through a tree right now (use smgx_submit_tokens)");
        if (n == 0) { *done_flag = done_value; return SMGX_SUCCESS; }
        const uint32_t cap = max_request_tokens ? std::min(max_request_tokens, P.cfg.max_tokens_per_request) : P.cfg.max_tokens_per_request;
        Lane& L = P.lanes[(P.mapped_seq++) % P.lanes.size()];   // any stream: nothing is staged, so a lane busy with a host-buffer submission is fine
        BatchDesc d{tokens, offsets, out_worker_idx, out_info, n, 0, nullptr};
        P.enqueue_batches(m, L, &d, 1, cap, done_flag, done_value);
        return SMGX_SUCCESS;
    });
}

smgx_status smgx_select_batch_tokens_device(smgx_policy* p, const char* model_key, uint32_t lane, const uint32_t* d_tokens,
                                            const uint32_t* d_offsets, uint32_t n, uint32_t max_request_tokens, int32_t* d_out_worker_idx,
                                            smgx_decision_info* d_out_info, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (d_tokens && d_offsets && d_out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(lane < P.lanes.size(), "lane out of range");
        ModelState& m = P.model(model_key, false);
        uint32_t cap = max_request_tokens ? std::min(max_request_tokens, P.cfg.max_tokens_per_request) : P.cfg.max_tokens_per_request;
        if (n) P.enqueue_tokens(m, P.lanes[lane], d_tokens, d_offsets, n, cap, d_out_worker_idx, d_out_info);
        return SMGX_SUCCESS;
    });
}

smgx_status smgx_select_many_tokens_device(smgx_policy* p, const char* model_key, uint32_t n_batches, const uint32_t* const* d_tokens,
                                           const uint32_t* const* d_offsets, const uint32_t* n, uint32_t max_request_tokens,
                                           int32_t* const* d_out_worker_idx, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n_batches == 0 || (d_tokens && d_offsets && n && d_out_worker_idx), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        uint32_t cap = max_request_tokens ? std::min(max_request_tokens, P.cfg.max_tokens_per_request) : P.cfg.max_tokens_per_request;
        if (n_batches >= 2 && n_batches <= 4096) {   // split path: hash stream and searches pipelined over two lanes
            std::vector<BatchDesc> all(n_batches);
            for (uint32_t k = 0; k < n_batches; ++k) all[k] = BatchDesc{d_tokens[k], d_offsets[k], d_out_worker_idx[k], nullptr, n[k], 0, nullptr};
            if (P.enqueue_split_pipelined(m, all.data(), n_batches, cap)) return SMGX_SUCCESS;
        }
        // up to kMaxMultiBatches batches per launch (blockIdx.y = batch); chunks alternate over the stream lanes
        // SMGX_SPREAD=1 (experiment): a short call is cut into one chunk per lane.  Measured worse than one launch pair:
        // small kernels run below the bandwidth a single large hash stream reaches.
        static const int spread = [] { const char* e = getenv("SMGX_SPREAD"); return e ? atoi(e) : 0; }();
        const uint32_t n_lanes = (uint32_t)P.lanes.size();
        const uint32_t per = spread ? std::min<uint32_t>(kMaxMultiBatches, std::max<uint32_t>(1, (n_batches + n_lanes - 1) / n_lanes)) : kMaxMultiBatches;
        uint32_t chunk_no = 0;
        for (uint32_t j0 = 0; j0 < n_batches; j0 += per, ++chunk_no) {
            BatchDesc d[kMaxMultiBatches];
            uint32_t cnt = std::min<uint32_t>(per, n_batches - j0);
            for (uint32_t k = 0; k < cnt; ++k) d[k] = BatchDesc{d_tokens[j0 + k], d_offsets[j0 + k], d_out_worker_idx[j0 + k], nullptr, n[j0 + k], 0, nullptr};
            P.enqueue_batches(m, P.lanes[chunk_no % P.lanes.size()], d, cnt, cap);
        }
        return SMGX_SUCCESS;
    });
}

smgx_status smgx_shard_candidates_device(smgx_policy* p, const char* model_key, uint32_t lane, const uint32_t* d_tokens, const uint32_t* d_offsets,
                                         uint32_t n, uint32_t max_request_tokens, smgx_shard_candidate* d_out_cand, smgx_shard_fleet* d_out_fleet,
                                         char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(d_out_cand); NONNULL(d_out_fleet);
        SMGX_REQUIRE(n == 0 || (d_tokens && d_offsets), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(lane < P.lanes.size(), "lane out of range");
        ModelState& m = P.model(model_key, false);
        uint32_t cap = max_request_tokens ? std::min(max_request_tokens, P.cfg.max_tokens_per_request) : P.cfg.max_tokens_per_request;
        Lane& L = P.lanes[lane];
        if (n) {
            BatchDesc d{d_tokens, d_offsets, nullptr, nullptr, n, 0, d_out_cand};
            P.enqueue_batches(m, L, &d, 1, cap);
        }
        // the shard's select_worker prologue, as computed by fleet_prepare_kernel for this fleet snapshot
        SMGX_CUDA(cudaMemcpyAsync(d_out_fleet, m.d_derived.ptr, sizeof(smgx_shard_fleet), cudaMemcpyDeviceToDevice, L.stream));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_shard_reduce_device(smgx_policy* p, uint32_t lane, const smgx_shard_candidate* d_cands, const smgx_shard_fleet* d_fleets,
                                     const uint32_t* global_base, uint32_t world, uint32_t n, int32_t* d_out_worker_idx,
                                     smgx_decision_info* d_out_info, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(d_cands); NONNULL(d_fleets); NONNULL(global_base); NONNULL(d_out_worker_idx);
        SMGX_REQUIRE(world >= 1 && world <= 64, "world out of range");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(lane < P.lanes.size(), "lane out of range");
        Lane& L = P.lanes[lane];
        P.d_gbase.reserve(64 * 4);
        SMGX_CUDA(cudaMemcpyAsync(P.d_gbase.ptr, global_base, (size_t)world * 4, cudaMemcpyHostToDevice, L.stream));
        launch_shard_reduce(d_cands, d_fleets, P.d_gbase.as<uint32_t>(), world, n, P.cfg.balance_abs_threshold, P.cfg.balance_rel_threshold,
                            d_out_worker_idx, d_out_info, L.stream);
        ++P.launches;
        return SMGX_SUCCESS;
    });
}

// ---- peer-memory exchange for sharded fleets ----
smgx_status smgx_shard_exchange_create(smgx_policy* p, uint32_t world, uint32_t rank, uint32_t max_batch, uint8_t* out_handle, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_handle);
        SMGX_REQUIRE(world >= 1 && world <= 64 && rank < world && max_batch > 0, "bad exchange geometry");
        static_assert(sizeof(cudaIpcMemHandle_t) == SMGX_IPC_HANDLE_BYTES, "IPC handle size");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        auto& x = P.xch;
        SMGX_REQUIRE(x.world == 0, "exchange already created");
        x.world = world; x.rank = rank; x.max_batch = max_batch;
        auto up = [](size_t v) { return (v + 255) / 256 * 256; };
        x.flag_off = 0;
        x.fleet_off = up((size_t)world * 8);
        x.cand_off = x.fleet_off + up((size_t)world * Policy::Exchange::kFleetStride);
        x.cand_slot_bytes = ((size_t)max_batch + 31) / 32 * 32 * sizeof(smgx_shard_candidate);   // 32 candidates = 768 B: keeps slots 256 B aligned
        x.parity_stride = x.cand_off + (size_t)world * x.cand_slot_bytes;
        x.local.reserve(2 * x.parity_stride);
        SMGX_CUDA(cudaMemset(x.local.ptr, 0, 2 * x.parity_stride));
        x.d_bases.reserve(2 * 64 * sizeof(void*));
        x.d_cand.reserve((size_t)max_batch * sizeof(smgx_shard_candidate));
        x.d_fleet.reserve(64);
        x.d_arrive.reserve(64);
        x.d_gbase.reserve(64 * 4);
        SMGX_CUDA(cudaMemset(x.d_arrive.ptr, 0, 64));
        SMGX_CUDA(cudaDeviceSynchronize());
        cudaIpcMemHandle_t h;
        SMGX_CUDA(cudaIpcGetMemHandle(&h, x.local.ptr));
        memcpy(out_handle, &h, sizeof(h));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_shard_exchange_connect(smgx_policy* p, const uint8_t* handles, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(handles);
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        auto& x = P.xch;
        SMGX_REQUIRE(x.world > 0 && !x.connected, "create the exchange first (once)");
        x.peer.assign(x.world, nullptr);
        x.opened.assign(x.world, false);
        for (uint32_t q = 0; q < x.world; ++q) {
            if (q == x.rank) { x.peer[q] = x.local.as<uint8_t>(); continue; }
            cudaIpcMemHandle_t h;
            memcpy(&h, handles + (size_t)q * SMGX_IPC_HANDLE_BYTES, sizeof(h));
            void* ptr = nullptr;
            SMGX_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
            x.peer[q] = (uint8_t*)ptr;
            x.opened[q] = true;
        }
        std::vector<uint8_t*> bases(2 * 64, nullptr);   // [parity][rank]
        for (uint32_t par = 0; par < 2; ++par) for (uint32_t q = 0; q < x.world; ++q) bases[par * 64 + q] = x.peer[q] + par * x.parity_stride;
        SMGX_CUDA(cudaMemcpy(x.d_bases.ptr, bases.data(), bases.size() * sizeof(void*), cudaMemcpyHostToDevice));
        x.connected = true;
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_shard_select_fused_device(smgx_policy* p, const char* model_key, uint32_t lane, const uint32_t* d_tokens, const uint32_t* d_offsets,
                                           uint32_t n, uint32_t max_request_tokens, const uint32_t* global_base, int32_t* d_out_worker_idx,
                                           smgx_decision_info* d_out_info, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(global_base); NONNULL(d_out_worker_idx);
        SMGX_REQUIRE(n == 0 || (d_tokens && d_offsets), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        auto& x = P.xch;
        SMGX_REQUIRE(x.connected, "peer-memory exchange is not connected");
        SMGX_REQUIRE(n <= x.max_batch, "batch larger than the exchange was created for");
        SMGX_REQUIRE(lane < P.lanes.size(), "lane out of range");
        ModelState& m = P.model(model_key, false);
        const uint32_t cap = max_request_tokens ? std::min(max_request_tokens, P.cfg.max_tokens_per_request) : P.cfg.max_tokens_per_request;
        Lane& L = P.lanes[lane];
        if (!x.seq) SMGX_CUDA(cudaMemcpyAsync(x.d_gbase.ptr, global_base, (size_t)x.world * 4, cudaMemcpyHostToDevice, L.stream));
        const uint64_t seq = ++x.seq;
        const uint32_t par = (uint32_t)(seq & 1);
        if (n) {
            BatchDesc d{d_tokens, d_offsets, nullptr, nullptr, n, 0, x.d_cand.as<smgx_shard_candidate>()};
            P.enqueue_batches(m, L, &d, 1, cap);
        } else {
            EventIndexView ixv; FleetView fv;
            P.sync_state(m, &ixv, &fv);
        }
        // stream order on this lane: candidates → push into every rank's buffer + flag → wait for every rank's flag → merge
        launch_shard_push(x.d_cand.as<smgx_shard_candidate>(), n, m.d_derived.as<smgx_shard_fleet>(),
                          reinterpret_cast<uint8_t* const*>(x.d_bases.as<uint8_t*>() + par * 64), x.world, x.rank, x.cand_off, x.cand_slot_bytes, x.fleet_off,
                          Policy::Exchange::kFleetStride, x.flag_off, seq, x.d_arrive.as<uint32_t>(), L.stream);
        launch_shard_reduce_wait(x.local.as<uint8_t>() + par * x.parity_stride, x.cand_off, (uint32_t)(x.cand_slot_bytes / sizeof(smgx_shard_candidate)),
                                 x.fleet_off, Policy::Exchange::kFleetStride, x.flag_off, seq, x.d_gbase.as<uint32_t>(), x.world, n,
                                 P.cfg.balance_abs_threshold, P.cfg.balance_rel_threshold, d_out_worker_idx, d_out_info, P.d_err.as<uint32_t>(), L.stream);
        P.launches += 2;
        SMGX_CUDA(cudaEventRecord(L.done, L.stream));
        L.has_done = true;
        return SMGX_SUCCESS;
    });
}

void* smgx_device_alloc(smgx_policy* p, size_t bytes, char** err) {
    void* out = nullptr;
    guard(err, [&]() {
        NONNULL(p);
        p->impl.use_device();
        SMGX_CUDA(cudaMalloc(&out, bytes ? bytes : 1));
        return SMGX_SUCCESS;
    });
    return out;
}
void smgx_device_free(smgx_policy* p, void* dptr) {
    if (p && dptr && p->impl.cfg.device_id >= 0) { cudaSetDevice(p->impl.cfg.device_id); cudaFree(dptr); }
}
smgx_status smgx_memcpy_h2d(smgx_policy* p, void* dptr, const void* host, size_t bytes, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(dptr); NONNULL(host);
        p->impl.use_device();
        SMGX_CUDA(cudaMemcpy(dptr, host, bytes, cudaMemcpyHostToDevice));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_memcpy_d2h(smgx_policy* p, void* host, const void* dptr, size_t bytes, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(dptr); NONNULL(host);
        p->impl.use_device();
        SMGX_CUDA(cudaMemcpy(host, dptr, bytes, cudaMemcpyDeviceToHost));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_synchronize(smgx_policy* p, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        p->impl.use_device();
        SMGX_CUDA(cudaDeviceSynchronize());
        uint32_t flag = 0;
        SMGX_CUDA(cudaMemcpy(&flag, p->impl.d_err.ptr, 4, cudaMemcpyDeviceToHost));
        if (flag) {
            SMGX_CUDA(cudaMemset(p->impl.d_err.ptr, 0, 4));
            if (flag & kErrNoSlowKernel)   // OR-ed into the flag (the lane and warp kernels OR their over-the-cap 1 as well), checked first
                throw Error(SMGX_UNKNOWN_ERROR, "internal error: a request needed event_slow_kernel in a launch that did not run it");
            if (flag == 2) throw Error(SMGX_DEVICE_ERROR, "peer-memory exchange: a rank did not publish its candidates in time");
            if (flag == 3) throw Error(SMGX_DEVICE_ERROR, "concurrent split launch: the search kernel gave up waiting for the hash kernel");
            throw Error(SMGX_INVALID_ARGUMENT, "a request exceeded max_tokens_per_request on the device-resident path");
        }
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_timer_start(smgx_policy* p, uint32_t lane, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        p->impl.use_device();
        SMGX_REQUIRE(lane < p->impl.lanes.size(), "lane out of range");
        SMGX_CUDA(cudaEventRecord(p->impl.lanes[lane].t0, p->impl.lanes[lane].stream));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_timer_stop_ms(smgx_policy* p, uint32_t lane, float* out_ms, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_ms);
        p->impl.use_device();
        SMGX_REQUIRE(lane < p->impl.lanes.size(), "lane out of range");
        Lane& l = p->impl.lanes[lane];
        SMGX_CUDA(cudaEventRecord(l.t1, l.stream));
        SMGX_CUDA(cudaEventSynchronize(l.t1));
        SMGX_CUDA(cudaEventElapsedTime(out_ms, l.t0, l.t1));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_timer_start_all(smgx_policy* p, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        Policy& P = p->impl;
        P.use_device();
        SMGX_CUDA(cudaEventRecord(P.lanes[0].t0, P.lanes[0].stream));
        for (size_t i = 1; i < P.lanes.size(); ++i) SMGX_CUDA(cudaStreamWaitEvent(P.lanes[i].stream, P.lanes[0].t0, 0));
        return SMGX_SUCCESS;
    });
}
// Same as smgx_timer_start_all, but a hold kernel first keeps lane 0 (and with it every lane, which waits for the start event) busy for
// ~hold_us microseconds: everything the caller enqueues in that window runs back to back once the hold ends, so the interval
// smgx_timer_stop_all_ms reports is GPU execution of the region, free of host launch latency.
smgx_status smgx_timer_start_all_gated(smgx_policy* p, uint32_t hold_us, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        Policy& P = p->impl;
        P.use_device();
        launch_hold(hold_us, P.lanes[0].stream);
        SMGX_CUDA(cudaEventRecord(P.lanes[0].t0, P.lanes[0].stream));
        for (size_t i = 1; i < P.lanes.size(); ++i) SMGX_CUDA(cudaStreamWaitEvent(P.lanes[i].stream, P.lanes[0].t0, 0));
        return SMGX_SUCCESS;
    });
}
// just the hold kernel on `lane` (bench.py: hold → untimed warm-up region → smgx_timer_start → timed region, all enqueued back to back)
smgx_status smgx_stream_hold(smgx_policy* p, uint32_t lane, uint32_t hold_us, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(lane < P.lanes.size(), "lane out of range");
        launch_hold(hold_us, P.lanes[lane].stream);
        return SMGX_SUCCESS;
    });
}
// single-lane form: hold kernel + start event on `lane`; pair with smgx_timer_stop_ms(lane)
smgx_status smgx_timer_start_gated(smgx_policy* p, uint32_t lane, uint32_t hold_us, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        Policy& P = p->impl;
        P.use_device();
        SMGX_REQUIRE(lane < P.lanes.size(), "lane out of range");
        launch_hold(hold_us, P.lanes[lane].stream);
        SMGX_CUDA(cudaEventRecord(P.lanes[lane].t0, P.lanes[lane].stream));
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_timer_stop_all_ms(smgx_policy* p, float* out_ms, char** err) {
    return guard(err, [&]() {
        NONNULL(p); NONNULL(out_ms);
        Policy& P = p->impl;
        P.use_device();
        for (size_t i = 1; i < P.lanes.size(); ++i) {
            SMGX_CUDA(cudaEventRecord(P.lanes[i].t1, P.lanes[i].stream));
            SMGX_CUDA(cudaStreamWaitEvent(P.lanes[0].stream, P.lanes[i].t1, 0));
        }
        SMGX_CUDA(cudaEventRecord(P.lanes[0].t1, P.lanes[0].stream));
        SMGX_CUDA(cudaEventSynchronize(P.lanes[0].t1));
        SMGX_CUDA(cudaEventElapsedTime(out_ms, P.lanes[0].t0, P.lanes[0].t1));
        return SMGX_SUCCESS;
    });
}
// ---- adjacent policy: power_of_two (model_gateway/src/policies/power_of_two.rs) ----
smgx_status smgx_power_of_two_update_loads(smgx_policy* p, const char* const* urls, const double* token_usage, uint32_t n, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (urls && token_usage), "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        for (uint32_t i = 0; i < n; ++i) { SMGX_REQUIRE(urls[i], "Invalid arguments: null pointer"); p->impl.p2c_usage[urls[i]] = token_usage[i]; }   // HashMap::extend (:130-134)
        return SMGX_SUCCESS;
    });
}
smgx_status smgx_power_of_two_select_batch(smgx_policy* p, const char* model_key, uint32_t n, uint64_t seed, int32_t* out_worker_idx, int32_t* out_pairs,
                                           uint8_t* out_metric, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || out_worker_idx, "Invalid arguments: null pointer");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        if (n == 0) return SMGX_SUCCESS;
        const uint32_t ns = (uint32_t)m.urls.size();
        SMGX_REQUIRE(m.loads.size() == ns && m.flags.size() == ns, "fleet state not set for this model (smgx_set_fleet_state)");
        std::vector<int32_t> healthy;
        std::vector<double> usage(std::max<uint32_t>(ns, 1), std::numeric_limits<double>::quiet_NaN());
        for (uint32_t i = 0; i < ns; ++i) {
            if ((m.flags[i] & 3) == 3) healthy.push_back((int32_t)i);   // is_healthy() && circuit_breaker_can_execute() (policies/mod.rs:137-144)
            auto it = P.p2c_usage.find(m.urls[i]);
            if (it != P.p2c_usage.end()) usage[i] = it->second;
        }
        Lane& lane = P.lanes[0];
        const size_t usage_bytes = usage.size() * 8, healthy_bytes = (std::max<size_t>(healthy.size(), 1) * 4 + 7) & ~(size_t)7, loads_bytes = (size_t)std::max<uint32_t>(ns, 1) * 8;
        P.scratch.reserve(usage_bytes + loads_bytes + healthy_bytes);
        P.scratch2.reserve((size_t)n * (4 + 8 + 1) + 16);
        double* d_usage = P.scratch.as<double>();
        uint64_t* d_loads = reinterpret_cast<uint64_t*>(d_usage + usage.size());
        int32_t* d_healthy = reinterpret_cast<int32_t*>(d_loads + std::max<uint32_t>(ns, 1));
        SMGX_CUDA(cudaMemcpyAsync(d_usage, usage.data(), usage_bytes, cudaMemcpyHostToDevice, lane.stream));
        if (ns) SMGX_CUDA(cudaMemcpyAsync(d_loads, m.loads.data(), (size_t)ns * 8, cudaMemcpyHostToDevice, lane.stream));
        if (!healthy.empty()) SMGX_CUDA(cudaMemcpyAsync(d_healthy, healthy.data(), healthy.size() * 4, cudaMemcpyHostToDevice, lane.stream));
        P2cArgs a;
        a.healthy = d_healthy; a.n_healthy = (uint32_t)healthy.size(); a.loads = d_loads; a.usage = d_usage; a.seed = seed; a.n = n;
        a.out_pair = reinterpret_cast<int32_t*>(P.scratch2.ptr);
        a.out_idx = a.out_pair + 2 * (size_t)n;
        a.out_metric = reinterpret_cast<uint8_t*>(a.out_idx + n);
        launch_power_of_two(a, lane.stream);
        ++P.launches;
        if (P.p2c_feedback) {
            SMGX_REQUIRE(ns <= kMaxP2cFeedbackSlice, "fleet too large for the load-feedback pass");
            launch_power_of_two_feedback(a, ns, lane.stream);
            ++P.launches;
        }
        SMGX_CUDA(cudaMemcpyAsync(out_worker_idx, a.out_idx, (size_t)n * 4, cudaMemcpyDeviceToHost, lane.stream));
        if (out_pairs) SMGX_CUDA(cudaMemcpyAsync(out_pairs, a.out_pair, (size_t)n * 8, cudaMemcpyDeviceToHost, lane.stream));
        if (out_metric) SMGX_CUDA(cudaMemcpyAsync(out_metric, a.out_metric, n, cudaMemcpyDeviceToHost, lane.stream));
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
        return SMGX_SUCCESS;
    });
}
// ---- adjacent policy: consistent_hashing (model_gateway/src/policies/consistent_hashing.rs) ----
smgx_status smgx_consistent_hashing_select_batch(smgx_policy* p, const char* model_key, uint32_t n, const uint8_t* values, const uint32_t* offsets,
                                                 const uint8_t* present, uint64_t seed, int32_t* out_worker_idx, uint8_t* out_branch,
                                                 uint64_t* out_key_pos, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        SMGX_REQUIRE(n == 0 || (offsets && present && out_worker_idx), "Invalid arguments: null pointer");
        SMGX_REQUIRE(n <= (0xFFFFFFFFu - 1) / kChashHeaders, "batch too large");
        std::lock_guard<std::mutex> g(p->impl.mu);
        Policy& P = p->impl;
        P.use_device();
        ModelState& m = P.model(model_key, false);
        if (n == 0) return SMGX_SUCCESS;
        const uint32_t ns = (uint32_t)m.urls.size();
        SMGX_REQUIRE(m.loads.size() == ns && m.flags.size() == ns, "fleet state not set for this model (smgx_set_fleet_state)");
        const uint32_t n_off = kChashHeaders * n + 1;
        uint32_t max_long = 0;
        for (uint32_t k = 0; k + 1 < n_off; ++k) {
            SMGX_REQUIRE(offsets[k + 1] >= offsets[k], "offsets must be non-decreasing");
            const uint32_t len = offsets[k + 1] - offsets[k], h = k % kChashHeaders;
            if (h == 0 || !((present[k / kChashHeaders] >> h) & 1)) continue;   // only a routing key or an implicit key is hashed
            SMGX_REQUIRE(len <= kChashMaxKeyBytes, "header value longer than 2 MiB");
            if (len > 1024) ++max_long;
        }
        const uint32_t base = offsets[0], bytes = offsets[n_off - 1] - base;
        SMGX_REQUIRE(bytes == 0 || values, "Invalid arguments: null pointer");
        // one pinned staging area, one copy: values | offsets rebased to 0 | present
        const size_t off_at = ((size_t)bytes + 15) & ~(size_t)15, pres_at = off_at + (size_t)n_off * 4;
        P.ch_stage.reserve(pres_at + n + 16);
        uint8_t* h_in = P.ch_stage.as<uint8_t>();
        if (bytes) memcpy(h_in, values + base, bytes);
        uint32_t* h_off = reinterpret_cast<uint32_t*>(h_in + off_at);
        for (uint32_t k = 0; k < n_off; ++k) h_off[k] = offsets[k] - base;
        memcpy(h_in + pres_at, present, n);
        Lane& lane = P.lanes[0];
        const size_t in_bytes = pres_at + n;
        lane.d_text.reserve(in_bytes + 16);
        SMGX_CUDA(cudaMemcpyAsync(lane.d_text.ptr, h_in, in_bytes, cudaMemcpyHostToDevice, lane.stream));
        RingView rv; PrefixFleetView fv;
        P.sync_chash(m, &rv, &fv);
        // outputs: key_pos (8n) | idx (4n) | branch (n), then the long-key queue (12n) and its length
        const size_t idx_at = (size_t)n * 8, br_at = idx_at + (size_t)n * 4, q_at = (br_at + n + 15) & ~(size_t)15;
        const size_t qlen_at = q_at + (size_t)n * sizeof(ChashLongKey);
        lane.d_out.reserve(qlen_at + 16);
        uint8_t* d_out = lane.d_out.as<uint8_t>();
        uint8_t* d_in = lane.d_text.as<uint8_t>();
        ChashArgs a;
        a.values = d_in; a.offsets = reinterpret_cast<const uint32_t*>(d_in + off_at); a.present = d_in + pres_at;
        a.n = n; a.seed = seed; a.ring = rv; a.fleet = fv;
        a.healthy = m.d_ch_lists.as<int32_t>(); a.n_healthy = m.ch_n_healthy;
        a.url_last = a.healthy + m.ch_n_healthy; a.n_url_last = (uint32_t)m.ch_lists.size() - m.ch_n_healthy;
        a.out_key_pos = reinterpret_cast<uint64_t*>(d_out); a.out_idx = reinterpret_cast<int32_t*>(d_out + idx_at); a.out_branch = d_out + br_at;
        a.queue = reinterpret_cast<ChashLongKey*>(d_out + q_at); a.queue_len = reinterpret_cast<uint32_t*>(d_out + qlen_at);
        P.launches += launch_consistent_hashing(a, max_long, P.sm_count, lane.stream);
        const size_t out_bytes = out_key_pos ? br_at + n : (out_branch ? (size_t)n * 5 : (size_t)n * 4);
        const size_t out_from = out_key_pos ? 0 : idx_at;
        P.ch_out.reserve(br_at + n + 16);
        uint8_t* h_out = P.ch_out.as<uint8_t>();
        SMGX_CUDA(cudaMemcpyAsync(h_out + out_from, d_out + out_from, out_bytes, cudaMemcpyDeviceToHost, lane.stream));
        SMGX_CUDA(cudaStreamSynchronize(lane.stream));
        memcpy(out_worker_idx, h_out + idx_at, (size_t)n * 4);
        if (out_branch) memcpy(out_branch, h_out + br_at, n);
        if (out_key_pos) memcpy(out_key_pos, h_out, (size_t)n * 8);
        return SMGX_SUCCESS;
    });
}

void smgx_set_event_path(int fused, int min_blocks_per_sm) {
    set_event_path(fused);
    if (min_blocks_per_sm) set_fused_minb(min_blocks_per_sm);
}
void smgx_set_fused_prefetch(int flavour) { set_fused_prefetch(flavour); }
void smgx_set_fused_tile(int tile, int64_t min_total) { set_fused_tile(tile, (long long)min_total); }
void smgx_set_event_simple(int min_blocks_per_sm) { set_event_simple(min_blocks_per_sm); }
void smgx_set_tile_depth(int depth) { set_tile_depth(depth); }
uint64_t smgx_kernel_launches(const smgx_policy* p) { return p ? p->impl.launches : 0; }
smgx_status smgx_flush_l2(smgx_policy* p, char** err) {
    return guard(err, [&]() {
        NONNULL(p);
        Policy& P = p->impl;
        P.use_device();
        size_t bytes = std::max<size_t>(P.l2_bytes * 2, 256u << 20);
        P.d_flush.reserve(bytes);
        launch_fill(P.d_flush.as<uint32_t>(), (uint32_t)P.launches, bytes / 4, P.lanes[0].stream);
        ++P.launches;
        return SMGX_SUCCESS;
    });
}

}  // extern "C"
