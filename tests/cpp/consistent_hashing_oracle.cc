/* ORACLE — test / bench infrastructure only.  Flat C surface over tests/cpp/consistent_hashing_oracle.h for ctypes
 * (tests/consistent_hashing_oracle.py): the packed header layout of smgx_consistent_hashing_select_batch, decided on host threads. */
#include <chrono>
#include <thread>

#include "consistent_hashing_oracle.h"

using namespace orc;

extern "C" {

void* chorc_ring_new(const char* const* urls, size_t n) {
    std::vector<std::string> u;
    for (size_t i = 0; i < n; ++i) u.emplace_back(urls[i]);
    return new HashRing(u);
}
void chorc_ring_free(void* r) { delete (HashRing*)r; }

// header h of request i = values[offsets[5i+h] .. offsets[5i+h+1]), present[i] bit h = get() returned Some; ring may be null (no ring).
// Request i uses draw i of `seed`.  The requests are split into `threads` contiguous shards decided on that many host threads.
// Returns the elapsed seconds of the decisions.
double chorc_select_batch(const char* const* urls, const uint8_t* healthy, size_t n_workers, const void* ring, const uint8_t* values,
                          const uint32_t* offsets, const uint8_t* present, size_t n, uint64_t seed, int threads, int32_t* out_idx,
                          uint8_t* out_branch, uint64_t* out_key_pos) {
    std::vector<ChWorker> ws(n_workers);
    for (size_t i = 0; i < n_workers; ++i) { ws[i].url = urls[i]; ws[i].healthy = healthy[i] != 0; }
    if (threads < 1) threads = 1;
    auto run = [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            ChHeaders h;
            for (int k = 0; k < 5; ++k)
                if ((present[i] >> k) & 1) h[k] = std::string((const char*)values + offsets[5 * i + k], offsets[5 * i + k + 1] - offsets[5 * i + k]);
            const ChDecision d = ConsistentHashingPolicy::select_worker(ws, (const HashRing*)ring, h, seed, i);
            out_idx[i] = (int32_t)d.idx;
            out_branch[i] = (uint8_t)d.branch;
            out_key_pos[i] = d.key_pos;
        }
    };
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; ++t) ts.emplace_back(run, n * (size_t)t / (size_t)threads, n * (size_t)(t + 1) / (size_t)threads);
    for (auto& th : ts) th.join();
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // extern "C"
