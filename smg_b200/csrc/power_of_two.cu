// power_of_two (policies/power_of_two.rs): "randomly selects two workers and routes to the one with lower load".
//
// The reference draws from a thread-local ChaCha generator nobody can seed (rand::rng(), :48), so there is no stream to be bit-equal
// to; what is reproduced is the procedure — idx1 uniform in 0..h, idx2 = (idx1 + 1 + uniform(0..h-1)) % h (:49-52), the metric rule
// (token usage only when BOTH candidates have a cached load response, otherwise request counts for both, :66-88) and the tie rule
// (load1 <= load2 keeps the first candidate, :91-95) — over a counter-based stream: draw k of a call is mix(seed + C·(k + 1)) with the
// splitmix64 finaliser, request i of the batch uses draws 2i and 2i + 1, and a draw x becomes an index as ⌊x·h / 2^64⌋.  The oracle
// (oracle/power_of_two.h) states the same stream independently; the GPU tests compare picks bit for bit.
#include "power_of_two.h"

#include "common.h"
#include "counter_draw.cuh"

namespace smgx {
namespace {

__global__ void __launch_bounds__(256) power_of_two_kernel(const P2cArgs a) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    int32_t out = -1, c1 = -1, c2 = -1;
    uint8_t metric = 2;
    const uint32_t h = a.n_healthy;
    if (h == 1) out = a.healthy[0];                                                    // :44-46
    else if (h >= 2) {
        const uint32_t i1 = (uint32_t)__umul64hi(p2c_draw(a.seed, 2ull * i), (uint64_t)h);
        const uint32_t i2 = (i1 + 1 + (uint32_t)__umul64hi(p2c_draw(a.seed, 2ull * i + 1), (uint64_t)(h - 1))) % h;   // never i1
        c1 = a.healthy[i1]; c2 = a.healthy[i2];
        const double u1 = a.usage[c1], u2 = a.usage[c2];
        const bool both = u1 == u1 && u2 == u2;                                         // neither is NaN: both workers have a cached load response
        const double l1 = both ? u1 : (double)a.loads[c1], l2 = both ? u2 : (double)a.loads[c2];
        metric = both ? 1 : 0;
        out = l1 <= l2 ? c1 : c2;                                                        // :91-95
    }
    a.out_idx[i] = out;
    if (a.out_pair) { a.out_pair[2 * i] = c1; a.out_pair[2 * i + 1] = c2; }
    if (a.out_metric) a.out_metric[i] = metric;
}

// Load feedback (smgx_set_load_feedback_policies, SMGX_FEEDBACK_POWER_OF_TWO): the gRPC router guards every pick (routers/grpc/context.rs:248-259),
// so request i compares loads that include the picks of requests < i.  The draws and the pairs do not depend on loads and come from
// power_of_two_kernel; this pass walks the requests in order with the running loads in shared memory and redoes the request-count
// comparison (metric 0: (double)load, first candidate on ties); token-usage comparisons and single-worker picks keep their result.  Then the
// pick's load is bumped.  The comparison chain is serial, so one thread walks it; the warp stages the loads.
__global__ void __launch_bounds__(32) power_of_two_feedback_kernel(const P2cArgs a, uint32_t n_slice) {
    extern __shared__ uint64_t s_L[];   // [n_slice]
    for (uint32_t i = threadIdx.x; i < n_slice; i += 32) s_L[i] = a.loads[i];
    __syncwarp();
    if (threadIdx.x != 0) return;
    for (uint32_t i = 0; i < a.n; ++i) {
        int32_t out = a.out_idx[i];
        if (a.out_metric[i] == 0) {
            const int32_t c1 = a.out_pair[2 * i], c2 = a.out_pair[2 * i + 1];
            out = (double)s_L[c1] <= (double)s_L[c2] ? c1 : c2;                          // :79-95
            a.out_idx[i] = out;
        }
        if (out >= 0) ++s_L[out];
    }
}

}  // namespace

void launch_power_of_two(const P2cArgs& a, cudaStream_t stream) {
    if (!a.n) return;
    power_of_two_kernel<<<(a.n + 255) / 256, 256, 0, stream>>>(a);
    SMGX_CUDA(cudaGetLastError());
}

void launch_power_of_two_feedback(const P2cArgs& a, uint32_t n_slice, cudaStream_t stream) {
    if (!a.n) return;
    const size_t smem = (size_t)(n_slice ? n_slice : 1) * 8;
    if (smem > 48 * 1024) SMGX_CUDA(cudaFuncSetAttribute(power_of_two_feedback_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    power_of_two_feedback_kernel<<<1, 32, smem, stream>>>(a, n_slice);
    SMGX_CUDA(cudaGetLastError());
}

}  // namespace smgx
