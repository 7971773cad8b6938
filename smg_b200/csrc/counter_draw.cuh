// The counter-based draw stream of the policies whose reference draws from rand::rng() (power_of_two, consistent_hashing's random
// fallback): draw k of the stream `seed` selects is the splitmix64 finaliser of seed + GOLDEN·(k + 1).  A draw x becomes an index of
// 0..h as ⌊x·h / 2^64⌋ (__umul64hi).
#pragma once
#include <cstdint>

namespace smgx {

__device__ __forceinline__ uint64_t p2c_mix(uint64_t x) {
    x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ULL;
    x ^= x >> 27; x *= 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t p2c_draw(uint64_t seed, uint64_t k) { return p2c_mix(seed + 0x9E3779B97F4A7C15ULL * (k + 1)); }

}  // namespace smgx
