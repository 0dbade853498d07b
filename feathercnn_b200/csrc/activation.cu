// ncnn's element-wise activation layers Sigmoid, TanH, Swish, HardSigmoid, HardSwish and GELU (fcuda_activation_forward).
//
// One flat grid-stride kernel per type, so the loop body is that type's arithmetic alone: float4 loads and stores where
// both pointers are 16-byte aligned, then a scalar tail.  Every rounding is written out (__fmul_rn / __fadd_rn /
// __fdiv_rn), so the compiler cannot contract x * alpha + beta into an FMA and the bits are those fcuda.h states.
#include "fcuda.h"

#include "activation.cuh"
#include "common.cuh"

#include <stdint.h>

namespace fcuda {

constexpr int kActThreads = 256;

struct HardParams {
    float alpha, beta, lower, upper;
};

template <int TYPE>
__device__ __forceinline__ float act_apply(float x, const HardParams& p) {
    if constexpr (TYPE == FCUDA_ACTIVATION_SIGMOID) {
        return sigm(x);
    } else if constexpr (TYPE == FCUDA_ACTIVATION_TANH) {
        return tanhf(x);
    } else if constexpr (TYPE == FCUDA_ACTIVATION_SWISH) {
        return __fdiv_rn(x, __fadd_rn(1.f, expf(-x)));
    } else if constexpr (TYPE == FCUDA_ACTIVATION_HARDSIGMOID) {
        // NaN fails both comparisons and reaches the linear branch, which propagates it
        return x < p.lower ? 0.f : x > p.upper ? 1.f : __fadd_rn(__fmul_rn(x, p.alpha), p.beta);
    } else if constexpr (TYPE == FCUDA_ACTIVATION_HARDSWISH) {
        return x < p.lower ? 0.f : x > p.upper ? x : __fmul_rn(x, __fadd_rn(__fmul_rn(x, p.alpha), p.beta));
    } else if constexpr (TYPE == FCUDA_ACTIVATION_GELU) {
        return __fmul_rn(__fmul_rn(0.5f, x), __fadd_rn(1.f, erff(__fmul_rn(x, 0.70710678118654752f))));
    } else {  // FCUDA_ACTIVATION_GELU_TANH
        const float x3 = __fmul_rn(__fmul_rn(x, x), x);
        const float z = __fmul_rn(0.79788456080286536f, __fadd_rn(x, __fmul_rn(0.044715f, x3)));
        return __fmul_rn(__fmul_rn(0.5f, x), __fadd_rn(1.f, tanhf(z)));
    }
}

// Plain loads: out may be in.
template <int TYPE>
__global__ void __launch_bounds__(kActThreads)
activation_kernel(float* out, const float* in, size_t n, HardParams p) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const bool vec = ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const size_t nv = vec ? n >> 2 : 0;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
        const float4 x = reinterpret_cast<const float4*>(in)[i];
        reinterpret_cast<float4*>(out)[i] = make_float4(act_apply<TYPE>(x.x, p), act_apply<TYPE>(x.y, p),
                                                        act_apply<TYPE>(x.z, p), act_apply<TYPE>(x.w, p));
    }
    for (size_t i = (nv << 2) + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = act_apply<TYPE>(in[i], p);
}

using ActKernel = void (*)(float*, const float*, size_t, HardParams);
constexpr ActKernel kActKernels[] = {activation_kernel<FCUDA_ACTIVATION_SIGMOID>, activation_kernel<FCUDA_ACTIVATION_TANH>,
                                     activation_kernel<FCUDA_ACTIVATION_SWISH>,
                                     activation_kernel<FCUDA_ACTIVATION_HARDSIGMOID>,
                                     activation_kernel<FCUDA_ACTIVATION_HARDSWISH>, nullptr,
                                     activation_kernel<FCUDA_ACTIVATION_GELU>,
                                     activation_kernel<FCUDA_ACTIVATION_GELU_TANH>};

int activation(float* out, const float* in, size_t n, int type, float alpha, float beta, float lower, float upper,
               cudaStream_t s) {
    const int prof = prof_begin(s, PROF_ACTIVATION, 0, 0, 8.0 * n);
    size_t blocks = ceil_div_sz(n / 4 + 1, kActThreads);
    const size_t cap = static_cast<size_t>(sm_count()) * 32;
    if (blocks > cap) blocks = cap;
    kActKernels[type]<<<static_cast<unsigned>(blocks), kActThreads, 0, s>>>(out, in, n,
                                                                           HardParams{alpha, beta, lower, upper});
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
