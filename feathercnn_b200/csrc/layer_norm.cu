// ncnn's LayerNorm (fcuda_layer_norm_forward): one warp per row, the rounding order fcuda.h states.
//
// Each lane walks its elements l, l + 32, ... in order, so the sums are the same whatever the row's alignment or the
// launch geometry.  Rows of at most 32 * kLnCache floats stay in registers between the passes (one read of the blob);
// longer rows (LayerNorm over a whole channel plane) are read again from global memory for each pass.
#include "fcuda.h"

#include "common.cuh"

namespace fcuda {

constexpr int kLnThreads = 256;
constexpr int kLnCache = 32;  // floats per lane kept in registers

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

template <bool CACHED>
__global__ void __launch_bounds__(kLnThreads)
layer_norm_kernel(float* out, const float* in, int n, long long rows, const float* gamma, const float* beta, float eps) {
    const int lane = threadIdx.x & 31;
    const long long warps = static_cast<long long>(gridDim.x) * (kLnThreads / 32);
    for (long long row = static_cast<long long>(blockIdx.x) * (kLnThreads / 32) + (threadIdx.x >> 5); row < rows;
         row += warps) {
        const float* x = in + row * n;
        float* y = out + row * n;
        float cache[CACHED ? kLnCache : 1];
        float s = 0.f;
        if constexpr (CACHED) {
#pragma unroll
            for (int j = 0; j < kLnCache; ++j) {
                const int i = lane + 32 * j;
                cache[j] = i < n ? x[i] : 0.f;
                if (i < n) s = __fadd_rn(s, cache[j]);
            }
        } else {
            for (int i = lane; i < n; i += 32) s = __fadd_rn(s, x[i]);
        }
        const float mean = __fdiv_rn(warp_sum(s), static_cast<float>(n));
        float q = 0.f;
        if constexpr (CACHED) {
#pragma unroll
            for (int j = 0; j < kLnCache; ++j) {
                const float d = __fsub_rn(cache[j], mean);
                if (lane + 32 * j < n) q = __fmaf_rn(d, d, q);
            }
        } else {
            for (int i = lane; i < n; i += 32) {
                const float d = __fsub_rn(x[i], mean);
                q = __fmaf_rn(d, d, q);
            }
        }
        const float var = __fdiv_rn(warp_sum(q), static_cast<float>(n));
        const float r = __frsqrt_rn(__fadd_rn(var, eps));
        // every lane has read its whole share of the row before any lane writes (output == input is allowed)
        __syncwarp();
        if constexpr (CACHED) {
#pragma unroll
            for (int j = 0; j < kLnCache; ++j) {
                const int i = lane + 32 * j;
                if (i >= n) break;
                const float t = __fmul_rn(__fsub_rn(cache[j], mean), r);
                y[i] = gamma ? __fmaf_rn(t, gamma[i], beta[i]) : t;
            }
        } else {
            for (int i = lane; i < n; i += 32) {
                const float t = __fmul_rn(__fsub_rn(x[i], mean), r);
                y[i] = gamma ? __fmaf_rn(t, gamma[i], beta[i]) : t;
            }
        }
    }
}

int layer_norm(float* out, const float* in, int n, long long rows, const float* gamma, const float* beta, float eps,
               cudaStream_t s) {
    const double bytes = 8.0 * n * static_cast<double>(rows) + (gamma ? 8.0 * n : 0.0);
    const int prof = prof_begin(s, PROF_LAYER_NORM, 0, 0, bytes);
    long long blocks = (rows + kLnThreads / 32 - 1) / (kLnThreads / 32);
    const long long cap = static_cast<long long>(sm_count()) * 16;
    if (blocks > cap) blocks = cap;
    if (n <= 32 * kLnCache)
        layer_norm_kernel<true><<<static_cast<unsigned>(blocks), kLnThreads, 0, s>>>(out, in, n, rows, gamma, beta, eps);
    else
        layer_norm_kernel<false><<<static_cast<unsigned>(blocks), kLnThreads, 0, s>>>(out, in, n, rows, gamma, beta, eps);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
