// Channel routing: ShuffleChannel, Slice and concatenation, alone or fused, as one gather.
//
// All three are pure copies.  ShuffleNet-v2 runs Concat -> ShuffleChannel -> Slice on the whole activation of a unit;
// one by one that is three reads and three writes of the blob in three launches (four with a two-bottom Concat), fused
// it is one read and one write in one launch.  Each thread owns a few output elements (float4s when every run of
// `inner` floats starts 16-byte aligned) and finds each one's source by arithmetic from the by-value RouteGeom: which destination and
// position it writes, the shuffled position that is, the concatenated position that came from, and the source holding
// it.  Nothing lives in device memory but the blobs, so the launch replays under CUDA graphs unchanged.  The index is
// flat over (image, outer, position, inner), so 7 x 7 planes fill warps as well as 56 x 56 ones; the divisions that
// split it and undo the shuffle are multiply-highs.
#include "common.cuh"
#include "route.cuh"

#include <stdint.h>

namespace fcuda {

constexpr int kRouteThreads = 256;
constexpr unsigned long long kRouteMaxUnits = 1ull << 31;  // output elements (or float4s) per launch

// floor(n / d) for n, d < 2^32 as the high half of n * m with m = ceil(2^64 / d); m == 0 stands for d == 1
static unsigned long long div_magic(unsigned long long d) { return d > 1 ? ~0ull / d + 1ull : 0ull; }
__device__ __forceinline__ unsigned fast_div(unsigned n, unsigned long long m) {
    return m ? static_cast<unsigned>(__umul64hi(n, m)) : n;
}

// Source and destination of output element e (T units: float4s when inner is counted in float4s)
template <class T>
__device__ __forceinline__ void route_locate(const RouteGeom& g, unsigned e, unsigned span, unsigned long long inner_m,
                                             unsigned long long span_m, unsigned long long g_m, const T*& src, T*& dst) {
    const unsigned row = fast_div(e, inner_m);
    const unsigned i = e - row * static_cast<unsigned>(g.inner);
    const unsigned bo = fast_div(row, span_m);  // image * outer + outer index
    const int m = static_cast<int>(row - bo * span);
    float* dp = g.dst[0];
    int db = 0, de = g.dst_begin[1];
#pragma unroll
    for (int k = 1; k < kRouteMax; ++k)
        if (k < g.num_dst && m >= g.dst_begin[k]) {
            dp = g.dst[k];
            db = g.dst_begin[k];
            de = g.dst_begin[k + 1] - db;
        }
    const unsigned p = static_cast<unsigned>(g.first + m);
    const unsigned q = fast_div(p, g_m);
    const int c = static_cast<int>((p - q * static_cast<unsigned>(g.g)) * static_cast<unsigned>(g.cpg) + q);
    const float* sp = g.src[0];
    int sb = 0, se = g.src_begin[1];
#pragma unroll
    for (int k = 1; k < kRouteMax; ++k)
        if (k < g.num_src && c >= g.src_begin[k]) {
            sp = g.src[k];
            sb = g.src_begin[k];
            se = g.src_begin[k + 1] - sb;
        }
    src = reinterpret_cast<const T*>(sp) + (static_cast<size_t>(bo) * se + (c - sb)) * g.inner + i;
    dst = reinterpret_cast<T*>(dp) + (static_cast<size_t>(bo) * de + (m - db)) * g.inner + i;
}

// T = float4 (inner counted in float4s) or float.  Each thread moves K elements kRouteThreads apart, all K loads issued
// before the stores.  The 4-byte path does the whole index computation for every float, the float4 path once per four:
// on 7 x 7 planes it reaches about a quarter of a device-to-device copy's rate, on 28 x 28 ones about 0.87 of it.
template <class T, int K>
__global__ void __launch_bounds__(kRouteThreads)
route_kernel(const RouteGeom g, unsigned span, unsigned long long inner_m, unsigned long long span_m,
             unsigned long long g_m, unsigned total) {
    const unsigned e0 = blockIdx.x * (kRouteThreads * K) + threadIdx.x;
    const T* src[K];
    T* dst[K];
    T v[K];
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (e0 + j * kRouteThreads < total) route_locate(g, e0 + j * kRouteThreads, span, inner_m, span_m, g_m, src[j], dst[j]);
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (e0 + j * kRouteThreads < total) v[j] = __ldg(src[j]);
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (e0 + j * kRouteThreads < total) *dst[j] = v[j];
}

int route_forward(const RouteGeom& geom, int batch, cudaStream_t s) {
    uintptr_t bits = 0;
    for (int k = 0; k < geom.num_src; ++k) bits |= reinterpret_cast<uintptr_t>(geom.src[k]);
    for (int k = 0; k < geom.num_dst; ++k) bits |= reinterpret_cast<uintptr_t>(geom.dst[k]);
    const int V = geom.inner % 4 == 0 && (bits & 15) == 0 ? 4 : 1;
    RouteGeom g = geom;
    g.inner = geom.inner / V;
    const unsigned span = static_cast<unsigned>(g.dst_begin[g.num_dst]);
    const unsigned long long per_image = static_cast<unsigned long long>(g.outer) * span * g.inner;  // < 2^31 (ABI)
    const unsigned long long inner_m = div_magic(g.inner), span_m = div_magic(span), g_m = div_magic(g.g);
    const int imgs = static_cast<int>(kRouteMaxUnits / per_image < static_cast<unsigned long long>(batch)
                                          ? kRouteMaxUnits / per_image : batch);
    const int prof = prof_begin(s, PROF_ROUTE, 0, 0, 8.0 * batch * static_cast<double>(per_image) * V);
    for (int n0 = 0; n0 < batch; n0 += imgs) {
        RouteGeom c = g;
        const size_t image = static_cast<size_t>(n0) * geom.outer * geom.inner;  // floats per position of n0 images
        for (int k = 0; k < g.num_src; ++k) c.src[k] = geom.src[k] + image * (g.src_begin[k + 1] - g.src_begin[k]);
        for (int k = 0; k < g.num_dst; ++k) c.dst[k] = geom.dst[k] + image * (g.dst_begin[k + 1] - g.dst_begin[k]);
        const int nb = batch - n0 < imgs ? batch - n0 : imgs;
        const unsigned total = static_cast<unsigned>(per_image * nb);
        const unsigned per_cta = kRouteThreads * (V == 4 ? 2 : 8);
        const unsigned blocks = static_cast<unsigned>((static_cast<unsigned long long>(total) + per_cta - 1) / per_cta);
        if (V == 4) route_kernel<float4, 2><<<blocks, kRouteThreads, 0, s>>>(c, span, inner_m, span_m, g_m, total);
        else route_kernel<float, 8><<<blocks, kRouteThreads, 0, s>>>(c, span, inner_m, span_m, g_m, total);
        FCUDA_CHECK_LAUNCH();
        count_launch();
    }
    prof_end(prof, s);
    return 0;
}

}  // namespace fcuda
