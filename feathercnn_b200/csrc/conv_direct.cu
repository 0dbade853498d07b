// NAIVE algorithm: fp32 CUDA-core implicit-GEMM convolution straight from NCHW.
//
// Device-side counterpart of NAIVE_Forward (/root/reference/src/booster/avx/booster.cpp:42-61: im2col +
// triple-loop GEMM + bias), which the reference authors used as their own oracle (ForceSelectAlgo(NAIVE)).
// Here it is the exact-fp32 second opinion for the tensor-core paths and the fallback for shapes TMA cannot
// describe.  64(oc) x 64(pixel) tile per block, K step 16, 4x4 outputs per thread; the B tile is gathered with
// the reference's im2col index rule (generic_kernels.cpp:66-67).
#include "conv_direct.cuh"
#include "common.cuh"

namespace fcuda {

template <bool CLIP>
__global__ void __launch_bounds__(256)
conv_direct_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                   float* __restrict__ out, PackGeom g, int OC, int act, float lo, float hi) {
    __shared__ float sW[16][64 + 4];
    __shared__ float sX[16][64 + 4];
    const int n = blockIdx.z;
    const int P = g.OH * g.OW;
    const int oc0 = blockIdx.y * 64, p0 = blockIdx.x * 64;
    const float* img = in + static_cast<size_t>(n) * g.IC * g.H * g.W;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int KHW = g.KH * g.KW;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < g.K; k0 += 16) {
        for (int i = threadIdx.x; i < 64 * 16; i += 256) {
            {   // weights: [oc][k], k fastest in memory
                const int r = i >> 4, c = i & 15;
                const int k = k0 + c;
                sW[c][r] = (oc0 + r < OC && k < g.K) ? __ldg(w + static_cast<size_t>(oc0 + r) * g.K + k) : 0.f;
            }
            {   // activations: pixel fastest so global reads are coalesced
                const int c = i >> 6, r = i & 63;
                const int k = k0 + c, pix = p0 + r;
                float v = 0.f;
                if (k < g.K && pix < P) {
                    const int ic = k / KHW, uv = k - ic * KHW;
                    const int u = uv / g.KW, vv = uv - u * g.KW;
                    const int oy = pix / g.OW, ox = pix - oy * g.OW;
                    const int iy = oy * g.stride_h - g.pad_top + u, ix = ox * g.stride_w - g.pad_left + vv;
                    if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
                        v = __ldg(img + (static_cast<size_t>(ic) * g.H + iy) * g.W + ix);
                }
                sX[c][r] = v;
            }
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = sW[c][ty * 4 + i]; b[i] = sX[c][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int oc = oc0 + ty * 4 + i;
        if (oc >= OC) continue;
        const float bv = bias ? __ldg(bias + oc) : 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int pix = p0 + tx * 4 + j;
            if (pix >= P) continue;
            float v = acc[i][j] + bv;
            if (act) v = act_clamp<CLIP>(v, lo, hi);
            out[(static_cast<size_t>(n) * OC + oc) * P + pix] = v;
        }
    }
}

int conv_direct(const float* in, const float* w, float* out, const PackGeom& g, int OC, const ConvEpilogue& e, int batch,
                cudaStream_t s) {
    dim3 grid(ceil_div(g.OH * g.OW, 64), ceil_div(OC, 64), batch);
    if (e.act == 2) conv_direct_kernel<true><<<grid, 256, 0, s>>>(in, w, e.bias, out, g, OC, e.act, e.lo, e.hi);
    else conv_direct_kernel<false><<<grid, 256, 0, s>>>(in, w, e.bias, out, g, OC, e.act, e.lo, e.hi);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
