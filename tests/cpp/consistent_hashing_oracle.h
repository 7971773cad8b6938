/* ORACLE — test / bench infrastructure only; never linked into the product.
 *
 * ConsistentHashingPolicy (model_gateway/src/policies/consistent_hashing.rs:53-196) restated line by line on the CPU, over the oracle's
 * own blake3 (oracle/blake3_ref.h) and HashRing (oracle/prefix_hash.h):
 *   1. an empty worker slice → (None, no_healthy_workers) before any header is read (:121-123);
 *   2. extract_header_value (routers/common/header_utils.rs:60-65): HeaderMap::get (the first value) → HeaderValue::to_str (every byte
 *      is \t or 0x20..=0x7E, the http crate's is_visible_ascii) → non-empty;
 *   3. X-SMG-Target-Worker, if extracted: usize::from_str (64-bit: optional '+', one or more ASCII digits, overflow is an error); a hit
 *      needs idx < len and is_healthy(), anything else is (None, target_worker_miss) (:128-137);
 *   4. X-SMG-Routing-Key, if extracted: find_by_consistent_hash → routing_key_hit, or (None, no_healthy_workers) (:139-145);
 *   5. the implicit key: the first PRESENT of authorization, x-forwarded-for, cookie; to_str and the non-empty filter come after that
 *      choice (:147-161);
 *   6. find_by_consistent_hash (:68-111): url → LAST healthy slice index (collect() overwrites; the circuit breaker is not read); an empty
 *      map → None; with a ring, find_healthy_url; without one, the sorted map values indexed by u64_le(blake3(key)[..8]) % len;
 *   7. the random fallback (:163-185): healthy_count over every is_healthy() worker, duplicates included; 0 → no_healthy_workers, else the
 *      random_range(0..healthy_count)-th healthy worker.  rand::rng() cannot be seeded, so request i of a batch uses draw i of the counter
 *      stream of oracle/power_of_two.h: x = splitmix64-finalise(seed + GOLDEN·(i + 1)), index ⌊x·h / 2^64⌋.
 * Pinned by tests/test_oracle_consistent_hashing.py (the reference's unit tests, one case per rule, goldens of the independent `blake3`
 * package) and compared there with the Python restatement tests/consistent_hashing_oracle.py.
 */
#pragma once
#include <array>
#include <cstdint>
#include <map>
#include <optional>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../oracle/power_of_two.h"
#include "../../oracle/prefix_hash.h"

namespace orc {

enum ChBranch { CH_NO_HEALTHY_WORKERS = 0, CH_TARGET_WORKER_HIT = 1, CH_TARGET_WORKER_MISS = 2, CH_ROUTING_KEY_HIT = 3, CH_RANDOM_FALLBACK = 4 };

// HeaderMap::get for x-smg-target-worker, x-smg-routing-key, authorization, x-forwarded-for, cookie; info.headers = None ⇔ all nullopt
using ChHeaders = std::array<std::optional<std::string>, 5>;

struct ChWorker { std::string url; bool healthy = true; };
struct ChDecision { int64_t idx = -1; ChBranch branch = CH_NO_HEALTHY_WORKERS; uint64_t key_pos = 0; };

class ConsistentHashingPolicy {
public:
    static const char* name() { return "consistent_hashing"; }   // :188-190

    static bool to_str_ok(const std::string& v) {                  // HeaderValue::to_str
        for (unsigned char c : v) if (!(c == '\t' || (c >= 0x20 && c <= 0x7E))) return false;
        return true;
    }
    static const std::string* extract(const std::optional<std::string>& v) {   // extract_header_value after get()
        return v && to_str_ok(*v) && !v->empty() ? &*v : nullptr;
    }
    static std::optional<uint64_t> parse_usize(const std::string& s) {   // <usize as FromStr>::from_str, 64-bit
        size_t k = !s.empty() && s[0] == '+' ? 1 : 0;
        if (k == s.size()) return std::nullopt;
        uint64_t v = 0;
        for (; k < s.size(); ++k) {
            const unsigned d = (unsigned char)s[k] - (unsigned)'0';
            if (d > 9 || v > (UINT64_MAX - d) / 10) return std::nullopt;
            v = v * 10 + d;
        }
        return v;
    }

    // :68-111
    static std::optional<size_t> find_by_consistent_hash(const std::vector<ChWorker>& ws, const HashRing* ring, const std::string& key) {
        std::unordered_map<std::string, size_t> healthy_url_to_idx;
        for (size_t i = 0; i < ws.size(); ++i) if (ws[i].healthy) healthy_url_to_idx[ws[i].url] = i;
        if (healthy_url_to_idx.empty()) return std::nullopt;
        if (ring) {
            const int64_t u = ring->find_healthy(key, [&](const std::string& url) { return healthy_url_to_idx.count(url) != 0; });
            if (u < 0) return std::nullopt;
            return healthy_url_to_idx[ring->url((size_t)u)];
        }
        std::vector<size_t> healthy_indices;
        for (auto& kv : healthy_url_to_idx) healthy_indices.push_back(kv.second);
        std::sort(healthy_indices.begin(), healthy_indices.end());
        return healthy_indices[(size_t)(HashRing::hash_position(key) % healthy_indices.size())];
    }

    // select_worker_impl (:116-180) for request i of a batch whose random draws come from `seed`
    static ChDecision select_worker(const std::vector<ChWorker>& ws, const HashRing* ring, const ChHeaders& h, uint64_t seed, uint64_t i) {
        ChDecision d;
        if (ws.empty()) return d;                                                            // :121-123
        if (const std::string* t = extract(h[0])) {                                          // :128-137
            const std::optional<uint64_t> idx = parse_usize(*t);
            if (idx && *idx < ws.size() && ws[*idx].healthy) { d.idx = (int64_t)*idx; d.branch = CH_TARGET_WORKER_HIT; }
            else d.branch = CH_TARGET_WORKER_MISS;
            return d;
        }
        const std::string* key = extract(h[1]);                                              // :139-145
        if (!key) {                                                                          // :147-155
            const std::optional<std::string>& first = h[2] ? h[2] : h[3] ? h[3] : h[4];
            key = extract(first);
        }
        if (key) {
            d.key_pos = HashRing::hash_position(*key);
            const std::optional<size_t> idx = find_by_consistent_hash(ws, ring, *key);
            if (idx) { d.idx = (int64_t)*idx; d.branch = CH_ROUTING_KEY_HIT; }
            return d;
        }
        size_t healthy_count = 0;                                                            // :163-167
        for (auto& w : ws) healthy_count += w.healthy ? 1 : 0;
        if (healthy_count == 0) return d;
        P2cStream rng(seed);
        rng.k = i;
        size_t nth = rng.random_range(healthy_count);                                        // :169-176
        for (size_t j = 0; j < ws.size(); ++j)
            if (ws[j].healthy && nth-- == 0) { d.idx = (int64_t)j; break; }
        d.branch = CH_RANDOM_FALLBACK;
        return d;
    }
};

}  // namespace orc
