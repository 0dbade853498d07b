// ncnn's Normalize: L2 normalisation of each pixel across its channels (SSD's conv4_3_norm), of each channel plane, or of
// the whole image, then a learned per-channel (or shared) scale.
//
// Per pixel (across_spatial 0), one launch.  A CTA owns `tp` consecutive pixels of one image (tp a power of two, 32 for
// C >= 256, up to 256 for small C) and loads the C channel rows of its tile from global into shared memory once, every
// load of the tile in flight together: 16-byte cp.async when plane % 4 == 0 and both blobs are 16-byte aligned, 4-byte
// cp.async otherwise.  Warp w sums the squares of channels w, w + 8, w + 16, ... of each pixel in increasing channel
// order (one fmaf per term); the eight warp partials of a pixel are then added in warp order, and the pixel's factor is
// computed once.  The tile is written back from shared memory, each channel row with coalesced (float4 where the loads
// were) stores.  So the blob crosses HBM once each way.  When C * tp * 4 bytes exceeds kStageBudget (C > 1024) the tile
// is not staged: the sums read it from global and the write pass re-reads it, from L2 in practice, with the same
// summation order.  Either way the result of a pixel depends on its C values only: not on the batch, the tile, the
// path or whether output == input.
//
// Across the image or a channel plane (across_spatial 1), two launches and no atomics.  The reduction set is a
// contiguous segment (the image, or one channel plane); CTA k of a segment sums the squares of its kSpatialChunk floats
// (each thread its strided elements in order, then a shuffle tree and the eight warp partials in order) into
// workspace[segment * K + k].  The second launch has the same CTAs: each adds its segment's K partials in a fixed order
// (lane-strided, then a shuffle tree), computes the factor and scales its chunk.
#include "common.cuh"
#include "normalize.cuh"

#include <stdint.h>

namespace fcuda {

namespace {

constexpr int kNormThreads = 256;
constexpr int kNormWarps = kNormThreads / 32;
constexpr int kMinTileShift = 5;                  // at least 32 pixels per CTA: one warp-wide row per channel
constexpr int kMaxTile = 256;                     // and at most 256
constexpr int kTileFloats = 8192;                 // tp grows while C * tp stays within this many floats
constexpr size_t kStageBudget = 128 * 1024;       // bytes of staged tile per CTA: C <= 1024 at tp = 32
constexpr int kSpatialChunk = 8192;               // floats per CTA in the across_spatial modes
constexpr long long kMaxBlocks = 0x7fffffffll;    // CTAs per launch

// The normalisation factor of a reduction set whose sum of squares is `ssum`, as fcuda.h states it per eps_mode.
__device__ __forceinline__ float norm_factor(float ssum, float eps, int mode) {
    if (mode == 0) return 1.f / sqrtf(ssum + eps);
    if (mode == 1) return 1.f / fmaxf(sqrtf(ssum), eps);
    return 1.f / sqrtf(fmaxf(ssum, eps));
}

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;"
                 ::"r"(static_cast<unsigned>(__cvta_generic_to_shared(smem_dst))), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;"
                 ::"r"(static_cast<unsigned>(__cvta_generic_to_shared(smem_dst))), "l"(gmem_src) : "memory");
}

// STAGE 0: the L2 fallback (sums and writes read global); 1: 4-byte staged tile; 2: 16-byte staged tile.
// Not __restrict__: output may equal input (each element is read, then written, by the same CTA).
template <int STAGE>
__global__ void __launch_bounds__(kNormThreads)
normalize_pixel_kernel(const float* in, float* out, const float* __restrict__ scale, int C, size_t plane, int shared,
                       int tp_shift, long long tiles, long long first_block, float eps, int eps_mode) {
    extern __shared__ float4 tile_smem[];
    float* tile = reinterpret_cast<float*>(tile_smem);
    __shared__ float red[kNormWarps][kMaxTile];
    __shared__ __align__(16) float factor[kMaxTile];
    const int tp = 1 << tp_shift;
    const long long b = first_block + blockIdx.x;
    const long long img = b / tiles;
    const size_t p0 = static_cast<size_t>(b - img * tiles) << tp_shift;
    const int np = plane - p0 < static_cast<size_t>(tp) ? static_cast<int>(plane - p0) : tp;
    const size_t base = static_cast<size_t>(img) * C * plane + p0;
    const float* x = in + base;
    float* y = out + base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    if (STAGE == 2) {  // plane % 4 == 0 and p0 % 32 == 0: np % 4 == 0 and every row segment 16-byte aligned
        const int q_shift = tp_shift - 2, nq = np >> 2;
        const int n = C << q_shift;
        for (int i = tid; i < n; i += kNormThreads) {
            const int c = i >> q_shift, j = i & ((1 << q_shift) - 1);
            if (j < nq) cp_async16(tile + (c << tp_shift) + 4 * j, x + static_cast<size_t>(c) * plane + 4 * j);
        }
    } else if (STAGE == 1) {
        const int n = C << tp_shift;
        for (int i = tid; i < n; i += kNormThreads) {
            const int c = i >> tp_shift, j = i & (tp - 1);
            if (j < np) cp_async4(tile + i, x + static_cast<size_t>(c) * plane + j);
        }
    }
    if (STAGE > 0) {
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();
    }

    // sum of squares per pixel: warp w takes channels w, w + 8, ... in order, then the warp partials in warp order
    for (int j = lane; j < tp; j += 32) {
        float s = 0.f;
        if (j < np) {
            for (int c = warp; c < C; c += kNormWarps) {
                const float v = STAGE > 0 ? tile[(c << tp_shift) + j] : x[static_cast<size_t>(c) * plane + j];
                s = fmaf(v, v, s);
            }
        }
        red[warp][j] = s;
    }
    __syncthreads();
    for (int j = tid; j < tp; j += kNormThreads) {
        float s = red[0][j];
#pragma unroll
        for (int w = 1; w < kNormWarps; ++w) s += red[w][j];
        factor[j] = norm_factor(s, eps, eps_mode);
    }
    __syncthreads();

    if (STAGE == 2) {
        const int q_shift = tp_shift - 2, nq = np >> 2;
        const int n = C << q_shift;
        for (int i = tid; i < n; i += kNormThreads) {
            const int c = i >> q_shift, j = i & ((1 << q_shift) - 1);
            if (j < nq) {
                const float sc = __ldg(scale + (shared ? 0 : c));
                const float4 v = *reinterpret_cast<const float4*>(tile + (c << tp_shift) + 4 * j);
                const float4 a = *reinterpret_cast<const float4*>(factor + 4 * j);
                *reinterpret_cast<float4*>(y + static_cast<size_t>(c) * plane + 4 * j) =
                    make_float4((v.x * a.x) * sc, (v.y * a.y) * sc, (v.z * a.z) * sc, (v.w * a.w) * sc);
            }
        }
    } else {
        const int n = C << tp_shift;
        for (int i = tid; i < n; i += kNormThreads) {
            const int c = i >> tp_shift, j = i & (tp - 1);
            if (j < np) {
                const float sc = __ldg(scale + (shared ? 0 : c));
                const size_t e = static_cast<size_t>(c) * plane + j;
                const float v = STAGE > 0 ? tile[i] : x[e];
                y[e] = (v * factor[j]) * sc;
            }
        }
    }
}

// Fixed-order block sum of one value per thread: a shuffle tree per warp, then the warp partials in warp order.
// The result is valid in thread 0.
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = red[0];
#pragma unroll
    for (int w = 1; w < kNormWarps; ++w) r += red[w];
    return r;
}

// Launch 1 of the across_spatial modes: partial[b] = sum of x^2 over chunk k of segment s (b = s * K + k).
__global__ void __launch_bounds__(kNormThreads)
normalize_partial_kernel(const float* in, float* __restrict__ partial, size_t seg_len, long long K, long long first_block) {
    __shared__ float red[kNormWarps];
    const long long b = first_block + blockIdx.x;
    const long long s = b / K, k = b - s * K;
    const size_t off = static_cast<size_t>(k) * kSpatialChunk;
    const size_t n = seg_len - off < static_cast<size_t>(kSpatialChunk) ? seg_len - off : kSpatialChunk;
    const float* x = in + static_cast<size_t>(s) * seg_len + off;
    float acc = 0.f;
    for (size_t i = threadIdx.x; i < n; i += kNormThreads) {
        const float v = x[i];
        acc = fmaf(v, v, acc);
    }
    const float r = block_sum(acc, red);
    if (threadIdx.x == 0) partial[b] = r;
}

// Launch 2: the segment's K partials in a fixed order, the factor, and the scaled chunk.  per_plane: the segment is one
// channel plane (channel s % C); otherwise the whole image (channel = offset / plane).
__global__ void __launch_bounds__(kNormThreads)
normalize_spatial_scale_kernel(const float* in, float* out, const float* __restrict__ partial,
                               const float* __restrict__ scale, size_t seg_len, long long K, int C, size_t plane,
                               int per_plane, int shared, float eps, int eps_mode, long long first_block) {
    __shared__ float a_sh;
    const long long b = first_block + blockIdx.x;
    const long long s = b / K, k = b - s * K;
    if (threadIdx.x < 32) {
        float r = 0.f;
        for (long long i = threadIdx.x; i < K; i += 32) r += partial[s * K + i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
        if (threadIdx.x == 0) a_sh = norm_factor(r, eps, eps_mode);
    }
    __syncthreads();
    const float a = a_sh;
    const size_t off = static_cast<size_t>(k) * kSpatialChunk;
    const size_t n = seg_len - off < static_cast<size_t>(kSpatialChunk) ? seg_len - off : kSpatialChunk;
    const size_t base = static_cast<size_t>(s) * seg_len + off;
    const int seg_c = per_plane ? static_cast<int>(s % C) : 0;
    for (size_t i = threadIdx.x; i < n; i += kNormThreads) {
        const int c = shared ? 0 : per_plane ? seg_c : static_cast<int>((off + i) / plane);
        out[base + i] = (in[base + i] * a) * __ldg(scale + c);
    }
}

// Pixels per CTA: a power of two in [32, kMaxTile] with C * tp <= kTileFloats where possible, no larger than
// the plane needs.
int pixel_tile_shift(int C, size_t plane) {
    int shift = kMinTileShift;
    while ((1 << shift) < kMaxTile && static_cast<long long>(C) << (shift + 1) <= kTileFloats &&
           (static_cast<size_t>(1) << shift) < plane)
        ++shift;
    return shift;
}

struct SpatialSplit {
    size_t seg_len;
    long long segments, K;
};
SpatialSplit spatial_split(int across_channel, int C, size_t plane, int batch) {
    SpatialSplit sp;
    sp.seg_len = across_channel ? static_cast<size_t>(C) * plane : plane;
    sp.segments = across_channel ? batch : static_cast<long long>(batch) * C;
    sp.K = static_cast<long long>(ceil_div_sz(sp.seg_len, kSpatialChunk));
    return sp;
}

}  // namespace

size_t normalize_workspace_floats(int across_spatial, int across_channel, int channels, size_t plane, int batch) {
    if (!across_spatial) return 0;
    const SpatialSplit sp = spatial_split(across_channel, channels, plane, batch);
    return static_cast<size_t>(sp.segments * sp.K);
}

int normalize_forward(const float* in, float* out, const float* scale, const NormalizeGeom& g, float* workspace,
                      cudaStream_t s) {
    const double n = static_cast<double>(g.batch) * g.channels * static_cast<double>(g.plane);
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, 8.0 * n + 4.0 * (g.shared ? 1 : g.channels));
    if (!g.across_spatial) {
        const int tp_shift = pixel_tile_shift(g.channels, g.plane);
        const size_t stage_bytes = static_cast<size_t>(g.channels) * sizeof(float) << tp_shift;
        const bool staged = stage_bytes <= kStageBudget;
        const bool wide = staged && g.plane % 4 == 0 &&
                          ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
        const long long tiles = static_cast<long long>((g.plane + (static_cast<size_t>(1) << tp_shift) - 1) >> tp_shift);
        const long long blocks = tiles * g.batch;
        const int smem = staged ? static_cast<int>(stage_bytes) : 0;
        static SmemAttrCache cache1, cache2;
        if (wide && ensure_dynamic_smem(normalize_pixel_kernel<2>, smem, cache2)) return FCUDA_ERR_CUDA;
        if (staged && !wide && ensure_dynamic_smem(normalize_pixel_kernel<1>, smem, cache1)) return FCUDA_ERR_CUDA;
        for (long long b0 = 0; b0 < blocks; b0 += kMaxBlocks) {
            const unsigned nb = static_cast<unsigned>(blocks - b0 < kMaxBlocks ? blocks - b0 : kMaxBlocks);
            if (wide)
                normalize_pixel_kernel<2><<<nb, kNormThreads, smem, s>>>(in, out, scale, g.channels, g.plane, g.shared,
                                                                         tp_shift, tiles, b0, g.eps, g.eps_mode);
            else if (staged)
                normalize_pixel_kernel<1><<<nb, kNormThreads, smem, s>>>(in, out, scale, g.channels, g.plane, g.shared,
                                                                         tp_shift, tiles, b0, g.eps, g.eps_mode);
            else
                normalize_pixel_kernel<0><<<nb, kNormThreads, 0, s>>>(in, out, scale, g.channels, g.plane, g.shared,
                                                                      tp_shift, tiles, b0, g.eps, g.eps_mode);
            FCUDA_CHECK_LAUNCH();
            count_launch();
        }
    } else {
        const SpatialSplit sp = spatial_split(g.across_channel, g.channels, g.plane, g.batch);
        const long long blocks = sp.segments * sp.K;
        for (long long b0 = 0; b0 < blocks; b0 += kMaxBlocks) {
            const unsigned nb = static_cast<unsigned>(blocks - b0 < kMaxBlocks ? blocks - b0 : kMaxBlocks);
            normalize_partial_kernel<<<nb, kNormThreads, 0, s>>>(in, workspace, sp.seg_len, sp.K, b0);
            FCUDA_CHECK_LAUNCH();
            count_launch();
        }
        for (long long b0 = 0; b0 < blocks; b0 += kMaxBlocks) {
            const unsigned nb = static_cast<unsigned>(blocks - b0 < kMaxBlocks ? blocks - b0 : kMaxBlocks);
            normalize_spatial_scale_kernel<<<nb, kNormThreads, 0, s>>>(in, out, workspace, scale, sp.seg_len, sp.K,
                                                                       g.channels, g.plane, !g.across_channel, g.shared,
                                                                       g.eps, g.eps_mode, b0);
            FCUDA_CHECK_LAUNCH();
            count_launch();
        }
    }
    prof_end(prof, s);
    return 0;
}

}  // namespace fcuda
