// smgx::ConsistentHashingPolicy (include/smgx.hpp) on the GPU: the reference's unit tests (consistent_hashing.rs:198-532) through the C++
// mirror, plus the header rules the mirror packs (case-insensitive names, first value of a repeated header, the implicit-key order).
#include <cstdio>
#include <functional>
#include <set>
#include <string>
#include <vector>

#include "../../include/smgx.hpp"

using namespace smgx;

static int g_tests = 0, g_failures = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_failures; } } while (0)

static Workers make(const std::vector<std::string>& urls) {
    Workers ws;
    for (auto& u : urls) ws.push_back(std::make_shared<BasicWorker>(u));
    return ws;
}
static BasicWorker& bw(const Workers& ws, size_t i) { return static_cast<BasicWorker&>(*ws[i]); }
static SelectWorkerInfo info(HeaderMap h, std::shared_ptr<HashRing> ring = nullptr) { SelectWorkerInfo i; i.headers = std::move(h); i.hash_ring = std::move(ring); return i; }
static void run(const char* name, const std::function<void()>& f) {
    ++g_tests;
    const int before = g_failures;
    try { f(); } catch (const std::exception& e) { std::printf("FAIL %s: %s\n", name, e.what()); ++g_failures; }
    std::printf("%s %s\n", g_failures == before ? "ok  " : "FAIL", name);
}

int main() {
    ConsistentHashingPolicy pol;
    const Workers w3 = make({"http://w1:8000", "http://w2:8000", "http://w3:8000"});
    const Workers w2 = make({"http://w1:8000", "http://w2:8000"});
    run("test_consistent_routing", [&] {
        auto first = pol.select_worker_impl(w3, info({{"x-smg-routing-key", "user-123"}}));
        CHECK(first.first.has_value() && first.second == SMGX_CH_ROUTING_KEY_HIT);
        for (int i = 0; i < 10; ++i) CHECK(pol.select_worker(w3, info({{"x-smg-routing-key", "user-123"}})) == first.first);
    });
    run("test_different_keys_distribute", [&] {
        std::set<size_t> d;
        for (int i = 0; i < 100; ++i) d.insert(*pol.select_worker(w3, info({{"x-smg-routing-key", "user-" + std::to_string(i)}})));
        CHECK(d.size() > 1);
    });
    run("test_target_worker_hit_miss_priority", [&] {
        CHECK(pol.select_worker_impl(w2, info({{"x-smg-target-worker", "1"}})).second == SMGX_CH_TARGET_WORKER_HIT);
        CHECK(pol.select_worker(w2, info({{"X-SMG-Target-Worker", "1"}})) == std::optional<size_t>(1));
        CHECK(pol.select_worker_impl(w2, info({{"x-smg-target-worker", "5"}})).second == SMGX_CH_TARGET_WORKER_MISS);
        CHECK(pol.select_worker(w2, info({{"x-smg-target-worker", "1"}, {"x-smg-routing-key", "some-key"}})) == std::optional<size_t>(1));
        const Workers u = make({"http://w1:8000", "http://w2:8000"});
        bw(u, 1).set_healthy(false);
        CHECK(pol.select_worker_impl(u, info({{"x-smg-target-worker", "1"}})).second == SMGX_CH_TARGET_WORKER_MISS);
    });
    run("test_fallback_random_distribution", [&] {
        std::set<size_t> d;
        for (int i = 0; i < 100; ++i) {
            auto r = pol.select_worker_impl(w3, SelectWorkerInfo());
            CHECK(r.first.has_value() && r.second == SMGX_CH_RANDOM_FALLBACK);
            if (r.first) d.insert(*r.first);
        }
        CHECK(d.size() > 1);
    });
    run("test_no_healthy_and_empty_workers", [&] {
        const Workers u = make({"http://w1:8000"});
        bw(u, 0).set_healthy(false);
        CHECK(pol.select_worker_impl(u, info({{"x-smg-routing-key", "test"}})).second == SMGX_CH_NO_HEALTHY_WORKERS);
        CHECK(!pol.select_worker(Workers{}, SelectWorkerInfo()).has_value());
    });
    run("test_consistent_hash_minimal_redistribution", [&] {
        const std::vector<std::string> urls = {"http://w0:8000", "http://w1:8000", "http://w2:8000", "http://w3:8000"};
        const Workers ws = make(urls);
        auto ring = pol.hash_ring(urls);
        std::vector<size_t> before;
        for (int i = 0; i < 100; ++i) before.push_back(*pol.select_worker(ws, info({{"x-smg-routing-key", "user-" + std::to_string(i)}}, ring)));
        bw(ws, 1).set_healthy(false);
        int moved = 0, on_failed = 0;
        for (int i = 0; i < 100; ++i) {
            const auto r = pol.select_worker(ws, info({{"x-smg-routing-key", "user-" + std::to_string(i)}}, ring));
            CHECK(r.has_value());
            moved += r != std::optional<size_t>(before[i]);
            on_failed += before[i] == 1;
        }
        CHECK(moved <= on_failed + 5 && moved < 50);
    });
    run("test_routing_key_failover_and_recovery", [&] {
        const Workers ws = make({"http://w0:8000", "http://w1:8000", "http://w2:8000"});
        auto ring = pol.hash_ring({"http://w0:8000", "http://w1:8000", "http://w2:8000"});
        const auto i = info({{"x-smg-routing-key", "session-abc-123"}}, ring);
        const size_t orig = *pol.select_worker(ws, i);
        bw(ws, orig).set_healthy(false);
        const auto fail = pol.select_worker(ws, i);
        CHECK(fail.has_value() && *fail != orig);
        for (int k = 0; k < 5; ++k) CHECK(pol.select_worker(ws, i) == fail);
        bw(ws, orig).set_healthy(true);
        CHECK(pol.select_worker(ws, i) == std::optional<size_t>(orig));
    });
    run("test_empty_routing_key_uses_fallback", [&] {
        CHECK(pol.select_worker_impl(w2, info({{"x-smg-routing-key", ""}})).second == SMGX_CH_RANDOM_FALLBACK);
    });
    run("test_implicit_key_order_and_first_value", [&] {
        auto key = [&](HeaderMap h) { return pol.select_worker_batch(w3, {std::optional<HeaderMap>(std::move(h))}).key_pos[0]; };
        const uint64_t xff = key({{"x-smg-routing-key", "10.0.0.1"}});
        CHECK(xff != 0 && key({{"X-Forwarded-For", "10.0.0.1"}, {"cookie", "c=1"}}) == xff);
        CHECK(key({{"x-forwarded-for", "10.0.0.1"}, {"x-forwarded-for", "10.0.0.2"}}) == xff);
        CHECK(pol.select_worker_impl(w3, info({{"authorization", ""}, {"x-forwarded-for", "10.0.0.1"}})).second == SMGX_CH_RANDOM_FALLBACK);
    });
    run("test_policy_name", [&] { CHECK(std::string(pol.name()) == "consistent_hashing"); });
    std::printf("%d tests, %d failures\n", g_tests, g_failures);
    return g_failures ? 1 : 0;
}
