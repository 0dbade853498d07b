// Shared helpers for the fcuda kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <math.h>
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

// What a convolution does to each output value after its contraction, in this order.  Built once per call by
// conv_epilogue() and handed to every kernel launcher; a launcher reads the fields its kernels have.
struct ConvEpilogue {
    const float* bias;      // OC floats or null
    const float* residual;  // fused Eltwise SUM (implicit GEMM only) or null
    int act;                // 0 none, 1 ReLU: fmaxf(v, 0), 2 Clip: fminf(fmaxf(v, lo), hi) in the Clip instantiations
    float lo, hi;
    int pool;               // 1: the output is the pooled (N, OC, (OH+1)/2, (OW+1)/2) blob (Winograd, implicit GEMM)
};

// `activation` is an FcudaActivation (the same numbering as `act`).  With a residual the convolution has no activation
// of its own and the one applied, after the sum, is the ReLU of relu_after_add.  Without Clip the bounds are [0, +inf],
// which stand for the ReLU where a kernel takes them at run time: fminf(fmaxf(v, 0), +inf) is fmaxf(v, 0) bit for bit,
// NaN included.
static inline ConvEpilogue conv_epilogue(int activation, bool bias_term, const float* bias, float clip_min, float clip_max,
                                         const float* residual, int relu_after_add, int pool) {
    ConvEpilogue e;
    e.bias = bias_term ? bias : nullptr;
    e.residual = residual;
    e.act = residual ? (relu_after_add ? 1 : 0) : (activation == 1 || activation == 2) ? activation : 0;
    e.lo = e.act == 2 ? clip_min : 0.f;
    e.hi = e.act == 2 ? clip_max : INFINITY;
    e.pool = pool ? 1 : 0;
    return e;
}

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
// The activation of the convolution epilogues: a Clip clamps to [lo, hi] (NaN -> lo); without CLIP it is the ReLU,
// fmaxf(v, 0).  The Clip kernels are instantiations of their own, so the ReLU kernels keep their code and registers.
template <bool CLIP>
__device__ __forceinline__ float act_clamp(float v, float lo, float hi) {
    return CLIP ? fminf(fmaxf(v, lo), hi) : fmaxf(v, 0.f);
}

__device__ __forceinline__ void split_tf32(float v, float& hi, float& lo) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));  // round to nearest (ties away), low 13 mantissa bits zero
    hi = __uint_as_float(r);
    lo = v - hi;
}

// Kernel-variant switches (defaults = the measured-best configuration; FCUDA_<NAME> in the environment or
// fcuda_set_tuning() override them — the variants stay testable and benchmarkable side by side).
enum TuneKey { TUNE_DW_VEC = 0, TUNE_IGEMM_HALO, TUNE_IGEMM_PRESPLIT, TUNE_IGEMM_WIDE, TUNE_IGEMM_STEM, TUNE_ROUTE_FUSE,
               TUNE_PERSISTENT_CTAS, TUNE_COUNT };
int tune_get(int key);
const char* tune_name(int key);             // registry name of a key (fcuda_set_tuning / fcuda_get_tuning)
int tune_set(const char* name, int value);  // 0, or -200 for an unknown name / value

// Grid of a persistent kernel: as many CTAs as fit on the device at once (occupancy x SMs), at most one per tile.  The
// switch persistent_ctas = n > 0 caps it at n CTAs, so tests can set how many tiles each CTA runs whatever the card.
template <class Kernel>
static inline int persistent_grid(Kernel kern, int threads, int smem, long long tiles, unsigned* grid) {
    int per_sm = 0;
    FCUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    long long slots = static_cast<long long>(sm_count()) * (per_sm > 0 ? per_sm : 1);
    const int cap = tune_get(TUNE_PERSISTENT_CTAS);
    if (cap > 0 && cap < slots) slots = cap;
    *grid = static_cast<unsigned>(tiles < slots ? tiles : slots);
    return 0;
}

// Per-launch profiling (tensor_gemm.cu): kernel classes for bench.py's roofline legs.
enum ProfKind { PROF_TENSOR_GEMM = 0, PROF_IGEMM = 1, PROF_WINO_INPUT = 2, PROF_WINO_OUTPUT = 3, PROF_POOL = 4,
                PROF_DEPTHWISE = 5, PROF_ELEMENTWISE = 6, PROF_DECONV = 7, PROF_RESIZE = 8, PROF_DETECTION = 9,
                PROF_ROUTE = 10, PROF_RCNN = 11, PROF_INSTANCE_NORM = 12, PROF_PIXEL_SHUFFLE = 13, PROF_ACTIVATION = 14,
                PROF_ATTENTION = 15, PROF_LAYER_NORM = 16, PROF_KINDS = 17 };
int prof_begin(cudaStream_t s, int kind, double algo_flops, double mma_flops, double algo_bytes);  // -1 when off
void prof_end(int idx, cudaStream_t s);
void profile_collect_kind(int kind, double* total_ms, double* algo_flops, double* mma_flops, double* algo_bytes,
                          long long* launches);

}  // namespace fcuda
