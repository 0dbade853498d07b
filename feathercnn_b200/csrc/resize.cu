// Interp (nearest / bilinear resize) and Crop, ncnn's layers of those names, for segmentation heads.
//
// Both are memory-bound, and an upsampling Interp is write-bound: x8 logits write 64 times the bytes they read.  A CTA
// of interp_kernel covers a band of output rows and up to 512 output columns of a plane.  It computes the source
// coordinates of its columns and rows once into shared memory, then each thread writes 4 consecutive outputs of a row
// as one float4 (when OW % 4 == 0) from input rows that the band's neighbours share in L1 / L2.  crop_kernel copies
// one output row per warp, with float4 accesses when the offsets and widths keep every row 16-byte aligned.
#include "common.cuh"
#include "resize.cuh"

#include <stdint.h>

namespace fcuda {

constexpr int kResizeThreads = 256;
constexpr int kResizeTileW = 512;    // output columns per CTA (12 bytes of shared coordinates each)
constexpr int kResizeMaxRows = 64;   // output rows per CTA
constexpr int kResizeItems = 2048;   // (row, column group) items per CTA and plane: 8 per thread
constexpr int kResizeMaxGridZ = 65535;
constexpr int kCropRowsPerCta = kResizeThreads / 32;

// Bilinear source coordinate of output index d: f = (d + 0.5) * scale - 0.5 clamped at 0, or d * scale with
// align_corner; the neighbours (int)f and min(i0 + 1, in - 1), and the weight f - i0 of the second one (exact in fp32).
__device__ __forceinline__ void bilinear_coord(int d, int in, float scale, int align, int& i0, int& i1, float& a) {
    float f = align ? __fmul_rn(static_cast<float>(d), scale)
                    : __fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(d), 0.5f), scale), 0.5f);
    f = fmaxf(f, 0.f);
    i0 = min(static_cast<int>(f), in - 1);
    i1 = min(i0 + 1, in - 1);
    a = f - static_cast<float>(i0);
}

template <int MODE, bool VEC>  // MODE 1 nearest, 2 bilinear; VEC: 4 outputs per thread, one float4 store
__global__ void __launch_bounds__(kResizeThreads)
interp_kernel(const float* __restrict__ in, float* __restrict__ out, InterpGeom g, int band, long long planes) {
    __shared__ int col0[kResizeTileW], col1[kResizeTileW];
    __shared__ float colw[kResizeTileW];
    __shared__ int row0[kResizeMaxRows], row1[kResizeMaxRows];
    __shared__ float roww[kResizeMaxRows];
    const int r_begin = blockIdx.x * band, rows = min(band, g.OH - r_begin);
    const int c_begin = blockIdx.y * kResizeTileW, cols = min(kResizeTileW, g.OW - c_begin);
    for (int i = threadIdx.x; i < cols; i += kResizeThreads) {
        if (MODE == 1) col0[i] = nearest_coord(c_begin + i, g.W, g.scale_w);
        else bilinear_coord(c_begin + i, g.W, g.scale_w, g.align_corner, col0[i], col1[i], colw[i]);
    }
    for (int i = threadIdx.x; i < rows; i += kResizeThreads) {
        if (MODE == 1) row0[i] = nearest_coord(r_begin + i, g.H, g.scale_h);
        else bilinear_coord(r_begin + i, g.H, g.scale_h, g.align_corner, row0[i], row1[i], roww[i]);
    }
    __syncthreads();
    constexpr int V = VEC ? 4 : 1;
    const int groups = cols / V;
    const int items = rows * groups;
    const size_t in_plane = static_cast<size_t>(g.H) * g.W, out_plane = static_cast<size_t>(g.OH) * g.OW;
    for (long long p = blockIdx.z; p < planes; p += gridDim.z) {
        const float* ip = in + static_cast<size_t>(p) * in_plane;
        float* op = out + static_cast<size_t>(p) * out_plane + static_cast<size_t>(r_begin) * g.OW + c_begin;
        for (int i = threadIdx.x; i < items; i += kResizeThreads) {
            const int r = i / groups, c = (i - r * groups) * V;
            float v[V];
            if (MODE == 1) {
                const float* src = ip + static_cast<size_t>(row0[r]) * g.W;
#pragma unroll
                for (int j = 0; j < V; ++j) v[j] = __ldg(src + col0[c + j]);
            } else {
                const float* s0 = ip + static_cast<size_t>(row0[r]) * g.W;
                const float* s1 = ip + static_cast<size_t>(row1[r]) * g.W;
                const float b = roww[r], b0 = 1.f - b;
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    const int x0 = col0[c + j], x1 = col1[c + j];
                    const float a = colw[c + j], a0 = 1.f - a;
                    // horizontally on both rows, then vertically: w0 * p + w1 * q as one product and one FMA each
                    const float h0 = fmaf(a, __ldg(s0 + x1), a0 * __ldg(s0 + x0));
                    const float h1 = fmaf(a, __ldg(s1 + x1), a0 * __ldg(s1 + x0));
                    v[j] = fmaf(b, h1, b0 * h0);
                }
            }
            float* dst = op + static_cast<size_t>(r) * g.OW + c;
            if constexpr (VEC) *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
            else dst[0] = v[0];
        }
    }
}

template <bool VEC>  // VEC: every source and destination row starts 16-byte aligned and OW % 4 == 0
__global__ void __launch_bounds__(kResizeThreads)
crop_kernel(const float* __restrict__ in, float* __restrict__ out, CropGeom g, long long rows) {
    const long long r = static_cast<long long>(blockIdx.x) * kCropRowsPerCta + (threadIdx.x >> 5);  // = (n, c, y)
    if (r >= rows) return;
    const int lane = threadIdx.x & 31;
    const long long plane = r / g.OH;
    const int y = static_cast<int>(r - plane * g.OH);
    const long long n = plane / g.OC;
    const int c = static_cast<int>(plane - n * g.OC);
    const float* src = in + ((static_cast<size_t>(n) * g.C + c + g.coff) * g.H + y + g.hoff) * g.W + g.woff;
    float* dst = out + static_cast<size_t>(r) * g.OW;
    if (VEC) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        const int n4 = g.OW >> 2;
#pragma unroll 4
        for (int x = lane; x < n4; x += 32) d4[x] = __ldg(s4 + x);
    } else {
        // 16 loads in flight per lane before the stores, as many bytes as the float4 path's unrolled loop
        constexpr int kInFlight = 16;
        for (int x0 = lane; x0 < g.OW; x0 += 32 * kInFlight) {
            float v[kInFlight];
#pragma unroll
            for (int k = 0; k < kInFlight; ++k)
                if (x0 + 32 * k < g.OW) v[k] = __ldg(src + x0 + 32 * k);
#pragma unroll
            for (int k = 0; k < kInFlight; ++k)
                if (x0 + 32 * k < g.OW) dst[x0 + 32 * k] = v[k];
        }
    }
}

int interp_forward(const float* in, float* out, const InterpGeom& g, long long planes, cudaStream_t s) {
    const double in_n = static_cast<double>(planes) * g.H * g.W, out_n = static_cast<double>(planes) * g.OH * g.OW;
    const int prof = prof_begin(s, PROF_RESIZE, 0, 0, 4.0 * (in_n + out_n));
    if (g.OH == g.H && g.OW == g.W && (g.mode == 2 || (g.scale_h == 1.f && g.scale_w == 1.f))) {
        // every source coordinate is the output index itself and every bilinear weight of the second neighbour is 0
        FCUDA_CHECK(cudaMemcpyAsync(out, in, static_cast<size_t>(out_n) * sizeof(float), cudaMemcpyDeviceToDevice, s));
    } else {
        const bool vec = g.OW % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
        const int groups = (g.OW < kResizeTileW ? g.OW : kResizeTileW) / (vec ? 4 : 1);
        int band = kResizeItems / groups;
        band = band < 1 ? 1 : (band > kResizeMaxRows ? kResizeMaxRows : band);
        const dim3 grid(static_cast<unsigned>(ceil_div(g.OH, band)), static_cast<unsigned>(ceil_div(g.OW, kResizeTileW)),
                        static_cast<unsigned>(planes < kResizeMaxGridZ ? planes : kResizeMaxGridZ));
        if (g.mode == 1) {
            if (vec) interp_kernel<1, true><<<grid, kResizeThreads, 0, s>>>(in, out, g, band, planes);
            else interp_kernel<1, false><<<grid, kResizeThreads, 0, s>>>(in, out, g, band, planes);
        } else {
            if (vec) interp_kernel<2, true><<<grid, kResizeThreads, 0, s>>>(in, out, g, band, planes);
            else interp_kernel<2, false><<<grid, kResizeThreads, 0, s>>>(in, out, g, band, planes);
        }
        FCUDA_CHECK_LAUNCH();
    }
    prof_end(prof, s);
    count_launch();
    return 0;
}

int crop_forward(const float* in, float* out, const CropGeom& g, int batch, cudaStream_t s) {
    const long long rows = static_cast<long long>(batch) * g.OC * g.OH;
    const long long blocks = (rows + kCropRowsPerCta - 1) / kCropRowsPerCta;
    if (blocks > 0x7fffffffLL) return -100;
    const bool vec = g.woff % 4 == 0 && g.W % 4 == 0 && g.OW % 4 == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    const int prof = prof_begin(s, PROF_RESIZE, 0, 0, 8.0 * rows * g.OW);
    if (vec) crop_kernel<true><<<static_cast<unsigned>(blocks), kResizeThreads, 0, s>>>(in, out, g, rows);
    else crop_kernel<false><<<static_cast<unsigned>(blocks), kResizeThreads, 0, s>>>(in, out, g, rows);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
