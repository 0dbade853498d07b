// ncnn's LRN: local response normalisation across channels (AlexNet, CaffeNet, GoogLeNet) or within each channel plane
// (Caffe's CIFAR-10 "full" model).  fcuda.h states the arithmetic; every product and sum below is an explicit
// __fmul_rn / __fadd_rn so that nvcc cannot contract `bias + a * ss` or `ss + v * v` into an fma.
//
// Across channels, one launch.  Each thread owns V consecutive pixels (V = 4: a 16-byte group, when plane % 4 == 0 and
// both pointers are 16-byte aligned; V = 1 otherwise) and walks the channels of its image.  The rows of the next
// kStages - 1 channels are in flight at once, each thread copying its own V floats into its own slots of a shared-memory
// ring with cp.async and waiting on its own commit groups, so no barrier is needed.  The thread keeps the values and
// squares of the last local_size channels in registers: the channel loop is unrolled by local_size, so every slot index
// is a compile-time constant.  Channel q is written once channel q + r has arrived; channels outside 0 .. C - 1 enter the
// window as squares of 0, which leave every partial sum unchanged (s + 0 == s for s >= 0), so the sum has the bits of
// the clipped window in ascending order.  Every input element crosses HBM once and every output element once.  Threads
// are numbered over (image, pixel group) of the whole batch, so a CTA may straddle two images and no CTA idles on a
// partial tile at the end of a plane.  local_size 1, 3, 5 and 7 are specialised; a larger size takes a generic kernel,
// one thread per output element, that reads its window through the cache.
//
// Within a channel, one launch.  A CTA owns a 32 x 16 tile of one plane; it squares the tile and its r-wide halo (clipped
// to the plane) once into shared memory, then each output adds the squares of its window row by row, skipping the terms
// outside the plane (they are 0).  When the clipped halo tile would exceed kWithinSmemBudget (local_size above about 85 on
// a large plane) the squares are read from global memory and recomputed in the same order instead.
#include "common.cuh"
#include "lrn.cuh"

#include <stdint.h>

namespace fcuda {

namespace {

constexpr int kAcrossThreads = 128;
constexpr int kStages = 8;                          // channel rows per thread in the ring; kStages - 1 in flight
constexpr int kGenericThreads = 256;
constexpr int kTileW = 32, kTileH = 16;             // within-channel output tile
constexpr int kWithinThreadsY = 8;                  // 32 x 8 threads, two rows each
constexpr int kWithinSmemBudget = 48 * 1024;        // bytes of halo tile: within the default dynamic limit
constexpr long long kMaxBlocks = 0x7fffffffll;      // CTAs per launch

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;"
                 ::"r"(static_cast<unsigned>(__cvta_generic_to_shared(smem_dst))), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;"
                 ::"r"(static_cast<unsigned>(__cvta_generic_to_shared(smem_dst))), "l"(gmem_src) : "memory");
}

// y = fl(x * powf(fl(bias + fl(a * ss)), -beta))
__device__ __forceinline__ float lrn_out(float x, float ss, float a, float bias, float nbeta) {
    return __fmul_rn(x, powf(__fadd_rn(bias, __fmul_rn(a, ss)), nbeta));
}

// Across channels, local_size L (odd, <= 7), V pixels per thread.  `groups` = batch * plane / V threads' worth of work.
template <int L, int V>
__global__ void __launch_bounds__(kAcrossThreads)
lrn_across_kernel(const float* __restrict__ in, float* __restrict__ out, int C, size_t plane, size_t groups_per_image,
                  size_t groups, long long first_block, float a, float bias, float nbeta) {
    constexpr int R = L / 2;
    __shared__ __align__(16) float ring[kStages][kAcrossThreads * V];
    const size_t g = static_cast<size_t>(first_block + blockIdx.x) * kAcrossThreads + threadIdx.x;
    if (g >= groups) return;  // the ring slots are this thread's own: no barrier below
    const size_t img = g / groups_per_image;
    const size_t base = img * C * plane + (g - img * groups_per_image) * V;
    const float* x = in + base;
    float* y = out + base;
    float* mine = &ring[0][threadIdx.x * V];
    auto fetch = [&](int c) {  // channel c's V floats into ring stage c % kStages, as one commit group
        if (c < C) {
            float* dst = mine + (c & (kStages - 1)) * (kAcrossThreads * V);
            if (V == 4) cp_async16(dst, x + static_cast<size_t>(c) * plane);
            else cp_async4(dst, x + static_cast<size_t>(c) * plane);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
#pragma unroll
    for (int c = 0; c < kStages - 1; ++c) fetch(c);

    float xs[L][V], sq[L][V];  // channel c sits in slot c % L
#pragma unroll
    for (int k = 0; k < L; ++k)
#pragma unroll
        for (int v = 0; v < V; ++v) xs[k][v] = sq[k][v] = 0.f;

    const int steps = C + R;  // step c brings channel c in and writes channel c - R
    for (int c0 = 0; c0 < steps; c0 += L) {
#pragma unroll
        for (int k = 0; k < L; ++k) {
            const int c = c0 + k;
            if (c >= steps) break;
            fetch(c + kStages - 1);
            asm volatile("cp.async.wait_group %0;" ::"n"(kStages - 1) : "memory");
            if (c < C) {
                const float* src = mine + (c & (kStages - 1)) * (kAcrossThreads * V);
                if (V == 4) {
                    const float4 t = *reinterpret_cast<const float4*>(src);
                    xs[k][0] = t.x;
                    xs[k][V > 1 ? 1 : 0] = t.y;
                    xs[k][V > 2 ? 2 : 0] = t.z;
                    xs[k][V > 3 ? 3 : 0] = t.w;
                } else {
                    xs[k][0] = src[0];
                }
#pragma unroll
                for (int v = 0; v < V; ++v) sq[k][v] = __fmul_rn(xs[k][v], xs[k][v]);
            } else {
#pragma unroll
                for (int v = 0; v < V; ++v) sq[k][v] = 0.f;
            }
            const int q = c - R;
            if (q >= 0) {
                float o[V];
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    float ss = sq[(k + 1) % L][v];  // channels q - R .. q + R: slots k + 1 .. k + L (mod L)
#pragma unroll
                    for (int t = 2; t <= L; ++t) ss = __fadd_rn(ss, sq[(k + t) % L][v]);
                    o[v] = lrn_out(xs[(k + R + 1) % L][v], ss, a, bias, nbeta);
                }
                float* dst = y + static_cast<size_t>(q) * plane;
                if (V == 4)
                    *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[V > 1 ? 1 : 0], o[V > 2 ? 2 : 0], o[V > 3 ? 3 : 0]);
                else
                    dst[0] = o[0];
            }
        }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
}

// Across channels, any odd local_size: one thread per output element, the window read through the cache.
__global__ void __launch_bounds__(kGenericThreads)
lrn_across_generic_kernel(const float* __restrict__ in, float* __restrict__ out, int C, size_t plane, size_t total,
                          long long first_block, int r, float a, float bias, float nbeta) {
    const size_t e = static_cast<size_t>(first_block + blockIdx.x) * kGenericThreads + threadIdx.x;
    if (e >= total) return;
    const size_t cp = e / plane;  // image * C + q
    const int q = static_cast<int>(cp % C);
    const float* col = in + (e - static_cast<size_t>(q) * plane);  // channel 0 of this pixel
    const int p0 = q - r < 0 ? 0 : q - r, p1 = q + r > C - 1 ? C - 1 : q + r;
    float ss = 0.f;
    for (int p = p0; p <= p1; ++p) {
        const float v = __ldg(col + static_cast<size_t>(p) * plane);
        ss = __fadd_rn(ss, __fmul_rn(v, v));
    }
    out[e] = lrn_out(__ldg(in + e), ss, a, bias, nbeta);
}

// Within a channel: one 32 x 16 output tile of one plane per CTA.  STAGED: the squares of the tile and its halo,
// clipped to the plane, in shared memory ((rows1 - rows0) x (cols1 - cols0) floats); otherwise recomputed from global.
template <bool STAGED>
__global__ void __launch_bounds__(kTileW * kWithinThreadsY)
lrn_within_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int r, int tiles_x,
                  long long tiles_per_plane, long long first_block, float a, float bias, float nbeta) {
    extern __shared__ float sqs[];
    const long long b = first_block + blockIdx.x;
    const long long nc = b / tiles_per_plane;
    const int t = static_cast<int>(b - nc * tiles_per_plane);
    const int i0 = t / tiles_x * kTileH, j0 = t % tiles_x * kTileW;
    const size_t off = static_cast<size_t>(nc) * H * W;
    const float* x = in + off;
    float* y = out + off;
    const int r0 = i0 - r < 0 ? 0 : i0 - r, r1 = i0 + kTileH + r < H ? i0 + kTileH + r : H;
    const int c0 = j0 - r < 0 ? 0 : j0 - r, c1 = j0 + kTileW + r < W ? j0 + kTileW + r : W;
    const int sw = c1 - c0;
    if (STAGED) {
        const int n = (r1 - r0) * sw;
        for (int e = threadIdx.y * kTileW + threadIdx.x; e < n; e += kTileW * kWithinThreadsY) {
            const int ri = e / sw;
            const float v = x[static_cast<size_t>(r0 + ri) * W + c0 + (e - ri * sw)];
            sqs[e] = __fmul_rn(v, v);
        }
        __syncthreads();
    }
    const int j = j0 + threadIdx.x;
    if (j >= W) return;
    const int dj0 = -r > -j ? -r : -j, dj1 = r < W - 1 - j ? r : W - 1 - j;
    for (int ii = threadIdx.y; ii < kTileH; ii += kWithinThreadsY) {
        const int i = i0 + ii;
        if (i >= H) break;
        const int di0 = -r > -i ? -r : -i, di1 = r < H - 1 - i ? r : H - 1 - i;
        float ss = 0.f;
        for (int di = di0; di <= di1; ++di) {
            for (int dj = dj0; dj <= dj1; ++dj) {
                float s;
                if (STAGED) {
                    s = sqs[(i + di - r0) * sw + (j + dj - c0)];
                } else {
                    const float v = x[static_cast<size_t>(i + di) * W + j + dj];
                    s = __fmul_rn(v, v);
                }
                ss = __fadd_rn(ss, s);
            }
        }
        const size_t e = static_cast<size_t>(i) * W + j;
        y[e] = lrn_out(x[e], ss, a, bias, nbeta);
    }
}

template <int L>
void launch_across(const float* in, float* out, const LrnGeom& g, bool wide, float a, float nbeta, cudaStream_t s) {
    const size_t plane = static_cast<size_t>(g.h) * g.w;
    const int V = wide ? 4 : 1;
    const size_t per_image = plane / V;
    const size_t groups = per_image * g.batch;
    const long long blocks = static_cast<long long>(ceil_div_sz(groups, kAcrossThreads));
    for (long long b0 = 0; b0 < blocks; b0 += kMaxBlocks) {
        const unsigned nb = static_cast<unsigned>(blocks - b0 < kMaxBlocks ? blocks - b0 : kMaxBlocks);
        if (wide)
            lrn_across_kernel<L, 4><<<nb, kAcrossThreads, 0, s>>>(in, out, g.channels, plane, per_image, groups, b0, a,
                                                                   g.bias, nbeta);
        else
            lrn_across_kernel<L, 1><<<nb, kAcrossThreads, 0, s>>>(in, out, g.channels, plane, per_image, groups, b0, a,
                                                                   g.bias, nbeta);
        count_launch();
    }
}

}  // namespace

int lrn_forward(const float* in, float* out, const LrnGeom& g, cudaStream_t s) {
    const size_t plane = static_cast<size_t>(g.h) * g.w;
    const size_t total = plane * g.channels * g.batch;
    const float nbeta = -g.beta;
    const int r = g.local_size / 2;
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, 8.0 * static_cast<double>(total));
    if (g.region == 0) {
        const float a = g.alpha / static_cast<float>(g.local_size);
        const bool wide = plane % 4 == 0 && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
        switch (g.local_size) {
            case 1: launch_across<1>(in, out, g, wide, a, nbeta, s); break;
            case 3: launch_across<3>(in, out, g, wide, a, nbeta, s); break;
            case 5: launch_across<5>(in, out, g, wide, a, nbeta, s); break;
            case 7: launch_across<7>(in, out, g, wide, a, nbeta, s); break;
            default: {
                const long long blocks = static_cast<long long>(ceil_div_sz(total, kGenericThreads));
                for (long long b0 = 0; b0 < blocks; b0 += kMaxBlocks) {
                    const unsigned nb = static_cast<unsigned>(blocks - b0 < kMaxBlocks ? blocks - b0 : kMaxBlocks);
                    lrn_across_generic_kernel<<<nb, kGenericThreads, 0, s>>>(in, out, g.channels, plane, total, b0, r, a,
                                                                              g.bias, nbeta);
                    count_launch();
                }
            }
        }
    } else {
        const float a = g.alpha / static_cast<float>(g.local_size * g.local_size);
        const int tiles_x = ceil_div(g.w, kTileW), tiles_y = ceil_div(g.h, kTileH);
        const long long per_plane = static_cast<long long>(tiles_x) * tiles_y;
        const long long blocks = per_plane * g.channels * g.batch;
        // the largest clipped halo tile of any CTA
        const long long rows = kTileH + 2ll * r < g.h ? kTileH + 2ll * r : g.h;
        const long long cols = kTileW + 2ll * r < g.w ? kTileW + 2ll * r : g.w;
        const long long smem = rows * cols * static_cast<long long>(sizeof(float));
        const bool staged = smem <= kWithinSmemBudget;
        const dim3 block(kTileW, kWithinThreadsY);
        for (long long b0 = 0; b0 < blocks; b0 += kMaxBlocks) {
            const unsigned nb = static_cast<unsigned>(blocks - b0 < kMaxBlocks ? blocks - b0 : kMaxBlocks);
            if (staged)
                lrn_within_kernel<true><<<nb, block, static_cast<int>(smem), s>>>(in, out, g.h, g.w, r, tiles_x,
                                                                                  per_plane, b0, a, g.bias, nbeta);
            else
                lrn_within_kernel<false><<<nb, block, 0, s>>>(in, out, g.h, g.w, r, tiles_x, per_plane, b0, a, g.bias,
                                                              nbeta);
            count_launch();
        }
    }
    const cudaError_t err = cudaGetLastError();
    prof_end(prof, s);
    return err == cudaSuccess ? 0 : FCUDA_ERR_CUDA;
}

}  // namespace fcuda
