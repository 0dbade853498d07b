// Operand packing kernels for the wgmma TensorGEMM.
//
//   im2col_pack   replaces booster::im2col (/root/reference/src/booster/avx/generic_kernels.cpp:50-85) and
//                 pack_B_avx (avx/sgemm.cpp:350-375): gathers the (ic,u,v) patch of every output pixel into a
//                 K-major row P[pixel][k] (k = (ic*KH + u)*KW + v, the reference's im2col row index), split into
//                 TF32 hi / fp32 lo planes.  Rows are zero-padded to Kp = round_up(K, 4) for TMA's 16-byte rule.
//   pack_weights  replaces packed_sgemm_init (avx/sgemm.cpp:312-346): W[oc][k] -> hi/lo planes padded to Kp.
//   split_tf32    elementwise hi/lo split (InnerProduct activations and weights).
//
// im2col_pack transposes through shared memory: global reads run along consecutive output pixels (coalesced for
// stride-1 layers), global writes along k (full 128-byte lines).
#include "pack.cuh"
#include "common.cuh"

namespace fcuda {

__global__ void __launch_bounds__(256)
im2col_pack_kernel(const float* __restrict__ in, float* __restrict__ P_hi, float* __restrict__ P_lo, PackGeom g,
                   long long m0, int rows) {
    __shared__ float tile[32][33];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r0 = blockIdx.x * 32;  // chunk-local first pixel row of this block

    // decode this lane's pixel once
    const long long m = m0 + r0 + lane;
    const bool m_ok = (r0 + lane) < rows;
    const int P = g.OH * g.OW;
    const int n = static_cast<int>(m / P);
    const int pix = static_cast<int>(m - static_cast<long long>(n) * P);
    const int oy = pix / g.OW, ox = pix - oy * g.OW;
    const int iy0 = oy * g.stride_h - g.pad_top, ix0 = ox * g.stride_w - g.pad_left;
    const float* img = in + static_cast<size_t>(n) * g.IC * g.H * g.W;
    const int KHW = g.KH * g.KW;

    for (int k0 = 0; k0 < g.Kp; k0 += 32) {
        // load: warp handles k = k0 + warp, +8, +16, +24 ; lane = pixel
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int kk = warp + i * 8;
            const int k = k0 + kk;
            float v = 0.f;
            if (m_ok && k < g.K) {
                const int ic = k / KHW;
                const int uv = k - ic * KHW;
                const int u = uv / g.KW, vv = uv - u * g.KW;
                const int iy = iy0 + u, ix = ix0 + vv;
                if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
                    v = __ldg(img + (static_cast<size_t>(ic) * g.H + iy) * g.W + ix);
            }
            tile[kk][lane] = v;
        }
        __syncthreads();
        // store: warp handles pixels warp, +8, +16, +24 ; lane = k
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int pr = warp + i * 8;
            const int k = k0 + lane;
            if (r0 + pr < rows && k < g.Kp) {
                const float v = tile[lane][pr];
                const size_t o = static_cast<size_t>(r0 + pr) * g.Kp + k;
                if (P_lo) {
                    float hi, lo;
                    split_tf32(v, hi, lo);
                    P_hi[o] = hi;
                    P_lo[o] = lo;
                } else {
                    P_hi[o] = v;
                }
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256)
pack_weights_kernel(const float* __restrict__ w, float* __restrict__ W_hi, float* __restrict__ W_lo, int rows, int K,
                    int Kp) {
    const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= static_cast<size_t>(rows) * Kp) return;
    const int r = static_cast<int>(idx / Kp), k = static_cast<int>(idx - static_cast<size_t>(r) * Kp);
    const float v = k < K ? w[static_cast<size_t>(r) * K + k] : 0.f;
    if (W_lo) {
        float hi, lo;
        split_tf32(v, hi, lo);
        W_hi[idx] = hi;
        W_lo[idx] = lo;
    } else {
        W_hi[idx] = v;
    }
}

__global__ void __launch_bounds__(256)
split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, size_t n) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float h, l;
        split_tf32(x[i], h, l);
        hi[i] = h;
        if (lo) lo[i] = l;
    }
}

int im2col_pack(const float* in, float* P_hi, float* P_lo, const PackGeom& g, long long m0, int rows,
                cudaStream_t s) {
    im2col_pack_kernel<<<ceil_div(rows, 32), 256, 0, s>>>(in, P_hi, P_lo, g, m0, rows);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int pack_weights(const float* w, float* W_hi, float* W_lo, int rows, int K, int Kp, cudaStream_t s) {
    const size_t total = static_cast<size_t>(rows) * Kp;
    pack_weights_kernel<<<static_cast<unsigned>(ceil_div_sz(total, 256)), 256, 0, s>>>(w, W_hi, W_lo, rows, K, Kp);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int split_tf32_planes(const float* x, float* hi, float* lo, size_t n, cudaStream_t s) {
    if (n == 0) return 0;
    size_t blocks = ceil_div_sz(n, 256);
    const size_t cap = static_cast<size_t>(sm_count()) * 16;
    if (blocks > cap) blocks = cap;
    split_tf32_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(x, hi, lo, n);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
