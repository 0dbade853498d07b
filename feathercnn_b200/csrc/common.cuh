// Shared helpers for the fcuda kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// Error convention mirrors the reference booster: 0 ok, negative int on failure
// (/root/reference/src/booster/avx/booster.cpp:306-307,349-353).  CUDA failures map to -700.
#define FCUDA_ERR_CUDA (-700)

#define FCUDA_CHECK(expr)                                                              \
    do {                                                                               \
        cudaError_t _e = (expr);                                                       \
        if (_e != cudaSuccess) {                                                       \
            fprintf(stderr, "fcuda: %s failed at %s:%d: %s\n", #expr, __FILE__,        \
                    __LINE__, cudaGetErrorString(_e));                                 \
            return FCUDA_ERR_CUDA;                                                     \
        }                                                                              \
    } while (0)

#define FCUDA_CHECK_LAUNCH() FCUDA_CHECK(cudaGetLastError())

namespace fcuda {

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline size_t ceil_div_sz(size_t a, size_t b) { return (a + b - 1) / b; }
static inline size_t round_up_sz(size_t a, size_t b) { return ceil_div_sz(a, b) * b; }

// Launch accounting for bench.py's gpu_launches (fcuda_launch_count).
void count_launch(int n = 1);
unsigned long long launch_count();
void reset_launch_count();

// Number of SMs of the current device (132 on H100 SXM); cached per device.
int sm_count();

// cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device): a process that drives several GPUs must opt
// in on each of them.  One cache object per call site (= per kernel instantiation), indexed by device ordinal.
constexpr int kMaxDevices = 64;
struct SmemAttrCache { int bytes[kMaxDevices] = {}; };
static inline int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) dev = 0;
    return dev < kMaxDevices ? dev : kMaxDevices - 1;
}
template <class Kernel>
static inline int ensure_dynamic_smem(Kernel kern, int bytes, SmemAttrCache& cache) {
    const int dev = current_device();
    if (bytes > cache.bytes[dev]) {
        FCUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        cache.bytes[dev] = bytes;
    }
    return 0;
}

// Split an fp32 value into a TF32-representable "hi" (round-to-nearest on the 13 dropped
// mantissa bits) and the exact fp32 remainder "lo".  hi + lo == v exactly; the tensor
// core then truncates lo to TF32, leaving a relative error of ~2^-22 per operand.
__device__ __forceinline__ void split_tf32(float v, float& hi, float& lo) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));  // round to nearest (ties away), low 13 mantissa bits zero
    hi = __uint_as_float(r);
    lo = v - hi;
}

// Kernel-variant switches (defaults = the measured-best configuration; FCUDA_<NAME> in the environment or
// fcuda_set_tuning() override them — the variants stay testable and benchmarkable side by side).
enum TuneKey { TUNE_DW_VEC = 0, TUNE_WINO_MLP, TUNE_IGEMM_HALO, TUNE_GEMM_PIPE, TUNE_IGEMM_PRESPLIT, TUNE_COUNT };
int tune_get(int key);
const char* tune_name(int key);             // registry name of a key (fcuda_set_tuning / fcuda_get_tuning)
int tune_set(const char* name, int value);  // 0, or -200 for an unknown name / value

// Per-launch profiling (tensor_gemm.cu): kernel classes for bench.py's roofline legs.
enum ProfKind { PROF_TENSOR_GEMM = 0, PROF_IGEMM = 1, PROF_WINO_INPUT = 2, PROF_WINO_OUTPUT = 3, PROF_POOL = 4,
                PROF_DEPTHWISE = 5, PROF_ELEMENTWISE = 6, PROF_DECONV = 7, PROF_KINDS = 8 };
int prof_begin(cudaStream_t s, int kind, double algo_flops, double mma_flops, double algo_bytes);  // -1 when off
void prof_end(int idx, cudaStream_t s);
void profile_collect_kind(int kind, double* total_ms, double* algo_flops, double* mma_flops, double* algo_bytes,
                          long long* launches);

}  // namespace fcuda
