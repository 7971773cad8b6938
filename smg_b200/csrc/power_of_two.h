// power_of_two policy (model_gateway/src/policies/power_of_two.rs:36-120) for a batch of requests: one thread per request.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace smgx {

struct P2cArgs {
    const int32_t* healthy;   // device [n_healthy]: get_healthy_worker_indices (policies/mod.rs:137-144) of the slice, in slice order
    uint32_t n_healthy;
    const uint64_t* loads;    // device [n_slice]: Worker::load()
    const double* usage;      // device [n_slice]: cached effective_token_usage() of the worker's URL, NaN = no cached load response
    uint64_t seed;            // the batch's draw stream (request i uses draws 2i and 2i + 1)
    uint32_t n;
    int32_t* out_idx;         // device [n]: slice index, -1 = None
    int32_t* out_pair;        // device [2n] or nullptr: the two candidates (-1, -1 when fewer than two healthy workers)
    uint8_t* out_metric;      // device [n] or nullptr: 0 = request_count, 1 = token_usage, 2 = no comparison made
};
void launch_power_of_two(const P2cArgs& a, cudaStream_t stream);
// load feedback: after launch_power_of_two, redo the request-count comparisons in request order on running loads (out_pair and out_metric
// must be set); the n_slice loads must fit in shared memory (kMaxP2cFeedbackSlice)
constexpr uint32_t kMaxP2cFeedbackSlice = 200 * 1024 / 8;
void launch_power_of_two_feedback(const P2cArgs& a, uint32_t n_slice, cudaStream_t stream);

}  // namespace smgx
