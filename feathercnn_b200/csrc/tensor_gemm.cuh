// TensorGEMM on Hopper warpgroup MMA — the replacement for the reference's 64-way batched "TensorGEMM"
// (avx/winograd_kernels_F63.cpp) and for its packed SGEMM (avx/sgemm.cpp).
//
//   for g in [0,G):   D_g[M x N] = A_g[M x K] * B_g[N x K]^T        (fp32 in, fp32 out)
//
// Both operands are K-major ("TN").  The contraction runs on the tensor cores as tf32 wgmma with fp32 accumulation in
// registers.  fp32 semantics are recovered with the 3xTF32 split (x = hi + lo exactly, hi TF32-representable): each
// k-step issues  A_lo*B_hi + A_hi*B_lo + A_hi*B_hi.
//   B (the small, reused operand: transformed filters / packed weights / FC activations) carries its hi and lo
//     planes in global memory (made once by the producer kernel);
//   A (the big streamed operand: Winograd V, im2col rows, FC weights) is stored ONCE as plain fp32: the kernel
//     lands the raw tile in shared memory by TMA and every consumer thread splits its own register fragment into
//     hi / lo, so A is one plane in HBM.
// planes == 1 runs plain TF32 (one MMA per k-step).
#pragma once

#include <cuda.h>

#include "common.cuh"

namespace fcuda {

enum GemmEpilogue : int {
    // D[g][m][n], n contiguous, row stride = ldd floats, batch stride = M*ldd.
    // Used for the Winograd product buffer M_e[tile][oc].
    EPI_ROWMAJOR = 0,
    // m = img * P + pix ;  out[(img * N + n) * P + pix] = act(acc + bias[n])      (NCHW conv output)
    EPI_NCHW = 1,
    // part[ks][n * ldd + m] = acc  — m = output feature, n = batch row (InnerProduct), ks = k-split index; plane stride
    // = split_stride floats.  Plain stores: the partial planes are summed in a fixed order by fc_reduce (layers.cu), so
    // the result does not depend on scheduling (round 1 used fp32 atomics here and was not run-to-run deterministic).
    EPI_COLMAJOR_PARTIAL = 2,
};

struct GemmProblem {
    // operands (device pointers)
    const float* A;                         // [G][M][K] plain fp32
    const float* B_hi; const float* B_lo;   // [G][N][K]; B_lo may be null when planes == 1
    float* D;
    int M, N, K, G;
    int planes;        // 1 = TF32, 2 = 3xTF32 (A split in-kernel, B_hi/B_lo planes)
    int epilogue;      // GemmEpilogue
    int ldd;           // EPI_ROWMAJOR / EPI_COLMAJOR_PARTIAL leading dimension (floats)
    int P;             // EPI_NCHW: pixels per image
    long long m_offset;  // EPI_NCHW: global pixel index of row 0 (chunked im2col); image = (m_offset + m) / P
    ConvEpilogue epi;  // EPI_NCHW: per-n bias and activation (bias, act, lo, hi; the other fields are not read)
    int split_k;       // >=1; only with EPI_COLMAJOR_PARTIAL
    long long split_stride;  // EPI_COLMAJOR_PARTIAL: floats between the partial planes of consecutive k-splits
    long long a_batch_stride;  // floats between consecutive g in A; 0 => dense (M*K)
    long long b_batch_stride;  // floats between consecutive g in B; 0 => dense (N*K)
    double algo_flops;         // algorithmic FLOPs this launch stands for (profiling only; 0 => 2*M*N*K*G)
};

// Launches the wgmma kernel on `stream`.  Returns 0 or a negative fcuda error.
// Requirements: K % 4 == 0, 16-byte aligned operand pointers.  M/N/K tails are zero-filled by TMA.
int tensor_gemm(const GemmProblem& p, cudaStream_t stream);

// Per-launch profiling of the TensorGEMM (bench.py's roofline leg): when enabled every tensor_gemm launch is
// bracketed by CUDA events on its own stream.  collect() synchronises and returns totals since enable.
void gemm_profile_enable(bool on);
void gemm_profile_collect(double* total_ms, double* algo_flops, double* mma_flops, long long* launches);

// Number of k-splits tensor_gemm will really use for (K, requested split): every split owns at least one 32-wide k-block.
int tensor_gemm_effective_split(int K, int split_k);

// True when the problem satisfies the TMA alignment rules above.
bool tensor_gemm_supported(const GemmProblem& p);

// cuTensorMapEncodeTiled, resolved once through the runtime (the library does not link libcuda); null without a driver.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn();

// K-major 3-D map over [G][rows][K] fp32 (batch_stride floats between consecutive g, 0 => rows * K) with a
// 32 x box_rows x 1 box and the 128-byte swizzle.  Returns 0 or FCUDA_ERR_CUDA.
int make_map(CUtensorMap* map, const float* base, int K, int rows, int G, long long batch_stride, int box_rows);

// Reference CUDA-core fp32 GEMM with identical semantics (used by the self-test and as
// the fallback for shapes TMA cannot describe).
int simt_gemm(const GemmProblem& p, cudaStream_t stream);

}  // namespace fcuda
