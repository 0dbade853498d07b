// ncnn's InstanceNorm (per-plane mean and biased variance, then an affine map), with the ReLU and a padding of the
// output plane fused into its write, and ncnn's Padding on its own.
//
// InstanceNorm takes two launches and no atomics.  Each (n, c) plane of S floats is cut into chunks of kChunk floats;
// CTA (plane, k) of launch 1 loads chunk k into registers (thread t owns elements 4t + 1024j + q, j = 0..7, q = 0..3,
// loaded as float4 when the plane and pointer allow, as floats otherwise: the same elements either way), sums it, and
// from the chunk mean m_k sums (x - m_k)^2 over the same registers.  It writes the chunk sum and the chunk-centred M2 to
// workspace[2 (plane K + k) + {0, 1}].  Launch 2 has one CTA per chunk of the *output* plane (padded or not): warp 0
// combines the plane's K partials in a fixed order by Chan's formula, M2 = sum M2_k + sum n_k (m_k - mean)^2, lane l
// taking chunks l, l + 32, ... then a 32-lane xor-shuffle tree, and computes a and b once; the CTA then writes its
// output chunk, each output element mapped to its source element by pad_src (the same index function as Padding).
// So a plane is read twice and written once, and its result depends on its own values only: the same bits for any
// batch split, pointer offset, in or out of place, eager or in a CUDA graph.  include/fcuda.h states the order.
#include "common.cuh"
#include "instance_norm.cuh"

#include <stdint.h>

namespace fcuda {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kQuads = 8;                               // float4 slots per thread
constexpr int kChunk = kThreads * 4 * kQuads;           // 8192 floats per CTA
constexpr long long kMaxBlocks = 0x7fffffffll;          // CTAs per launch

// Source index along one axis of a padded plane: output coordinate o (0 .. n + before + after - 1) of an axis of n
// elements, `before` of them added in front.  -1: a constant border.  reflect needs before, after < n.
__device__ __forceinline__ int pad_src(int o, int n, int before, int type) {
    const int i = o - before;
    if (i >= 0 && i < n) return i;
    if (type == 0) return -1;
    if (type == 1) return i < 0 ? 0 : n - 1;
    return i < 0 ? -i : 2 * (n - 1) - i;
}

// Fixed-order sum of one value per thread: a 32-lane xor-shuffle tree (every lane ends with the same bits), then the
// eight warp partials in warp order.  Every thread returns the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = red[0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) r += red[w];
    return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Launch 1: partial[2b] = sum of chunk k of plane p, partial[2b + 1] = sum of (x - m_k)^2 over it (b = p * K + k).
// VEC: S % 4 == 0 and `in` 16-byte aligned.
template <bool VEC>
__global__ void __launch_bounds__(kThreads)
instance_norm_stats_kernel(const float* in, float* __restrict__ partial, size_t S, long long K, long long first_block) {
    __shared__ float red0[kWarps], red1[kWarps];
    const long long b = first_block + blockIdx.x;
    const long long p = b / K, k = b - p * K;
    const size_t off = static_cast<size_t>(k) * kChunk;
    const int n = S - off < static_cast<size_t>(kChunk) ? static_cast<int>(S - off) : kChunk;
    const float* x = in + static_cast<size_t>(p) * S + off;
    const int t4 = 4 * threadIdx.x;
    float v[kQuads][4];
#pragma unroll
    for (int j = 0; j < kQuads; ++j) {
        const int e = 1024 * j + t4;
        if (VEC) {
            const float4 q = e < n ? __ldg(reinterpret_cast<const float4*>(x + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
            v[j][0] = q.x; v[j][1] = q.y; v[j][2] = q.z; v[j][3] = q.w;
        } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) v[j][q] = e + q < n ? __ldg(x + e + q) : 0.f;
        }
    }
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kQuads; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (1024 * j + t4 + q < n) s += v[j][q];
    const float sum = block_sum(s, red0);
    const float m = sum / static_cast<float>(n);
    float m2 = 0.f;
#pragma unroll
    for (int j = 0; j < kQuads; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (1024 * j + t4 + q < n) {
                const float d = v[j][q] - m;
                m2 = fmaf(d, d, m2);
            }
    const float M2 = block_sum(m2, red1);
    if (threadIdx.x == 0) {
        partial[2 * b] = sum;
        partial[2 * b + 1] = M2;
    }
}

struct Identity {
    __device__ __forceinline__ float operator()(float x) const { return x; }
};
struct Affine {
    float a, b;
    int relu;
    __device__ __forceinline__ float operator()(float x) const {
        const float y = fmaf(x, a, b);
        return relu ? fmaxf(y, 0.f) : y;  // the ReLU kernel's expression (layers.cu)
    }
};

// Writes output chunk `off` (n floats) of one plane: thread t the elements off + 4t + 1024j + q.  PAD: the output plane
// is Ho x Wo and each element comes from pad_src (constant borders take pad.value, untouched by op; y never aliases x);
// otherwise the element of the same index, which y may alias (each element is read, then written, by one thread).
// VEC: float4 stores (and, unpadded, float4 loads); needs So % 4 == 0 and 16-byte aligned planes.
template <bool PAD, bool VEC, class Op>
__device__ __forceinline__ void write_chunk(const float* x, float* y, size_t off, int n, int h, int w, int Wo,
                                            const PlanePad& pad, Op op) {
    const int t4 = 4 * threadIdx.x;
#pragma unroll 2
    for (int j = 0; j < kQuads; ++j) {
        const int e = 1024 * j + t4;
        if (e >= n) break;
        float r[4];
        if (!PAD) {  // y may alias x here: plain loads, not the read-only (.nc) path
            if (VEC) {
                const float4 q = *reinterpret_cast<const float4*>(x + off + e);
                r[0] = op(q.x); r[1] = op(q.y); r[2] = op(q.z); r[3] = op(q.w);
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q) r[q] = e + q < n ? op(x[off + e + q]) : 0.f;
            }
        } else {
            const size_t flat = off + e;
            int oy = static_cast<int>(flat / static_cast<unsigned>(Wo));
            int ox = static_cast<int>(flat - static_cast<size_t>(oy) * Wo);
            int sy = pad_src(oy, h, pad.top, pad.type);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int sx = pad_src(ox, w, pad.left, pad.type);
                r[q] = (sy < 0 || sx < 0 || e + q >= n) ? pad.value : op(__ldg(x + static_cast<size_t>(sy) * w + sx));
                if (++ox == Wo) {
                    ox = 0;
                    sy = pad_src(++oy, h, pad.top, pad.type);
                }
            }
        }
        if (VEC) {
            *reinterpret_cast<float4*>(y + off + e) = make_float4(r[0], r[1], r[2], r[3]);
        } else {
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (e + q < n) y[off + e + q] = r[q];
        }
    }
}

// Launch 2: CTA (plane p, output chunk k2) combines plane p's K partials (warp 0), then writes its output chunk.  Every
// CTA of a plane re-reads the K partials (K * K2 * 8 bytes per plane, from L2); the ABI caps the input and the padded
// plane at 2^24 floats, so that stays below 32 MB for a 64 MB plane.
// Not __restrict__: output may equal input when unpadded (each element is read, then written, by the same thread).
template <bool PAD, bool VEC>
__global__ void __launch_bounds__(kThreads)
instance_norm_apply_kernel(const float* in, float* out, const float* __restrict__ partial,
                           const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int relu, int C,
                           int h, int w, size_t S, long long K, int Wo, size_t So, long long K2, PlanePad pad,
                           long long first_block) {
    __shared__ float ab[2];
    const long long b = first_block + blockIdx.x;
    const long long p = b / K2, k2 = b - p * K2;
    if (threadIdx.x < 32) {
        const float* part = partial + 2 * p * K;
        float s = 0.f;
        for (long long i = threadIdx.x; i < K; i += 32) s += part[2 * i];
        const float mean = warp_sum(s) / static_cast<float>(S);
        float m2 = 0.f;
        for (long long i = threadIdx.x; i < K; i += 32) {
            const size_t o = static_cast<size_t>(i) * kChunk;
            const float nk = static_cast<float>(S - o < static_cast<size_t>(kChunk) ? S - o : kChunk);
            const float d = part[2 * i] / nk - mean;
            m2 += fmaf(nk * d, d, part[2 * i + 1]);
        }
        const float var = warp_sum(m2) / static_cast<float>(S);
        if (threadIdx.x == 0) {
            const int c = static_cast<int>(p % C);
            const float r = sqrtf(var + eps);
            const float a = gamma ? __ldg(gamma + c) / r : 1.f / r;
            ab[0] = a;
            ab[1] = fmaf(-mean, a, beta ? __ldg(beta + c) : 0.f);
        }
    }
    __syncthreads();
    const size_t off = static_cast<size_t>(k2) * kChunk;
    const int n = So - off < static_cast<size_t>(kChunk) ? static_cast<int>(So - off) : kChunk;
    write_chunk<PAD, VEC>(in + static_cast<size_t>(p) * S, out + static_cast<size_t>(p) * So, off, n, h, w, Wo, pad,
                          Affine{ab[0], ab[1], relu});
}

template <bool PAD, bool VEC>
__global__ void __launch_bounds__(kThreads)
padding_kernel(const float* in, float* out, int h, int w, size_t S, int Wo, size_t So, long long K2, PlanePad pad,
               long long first_block) {
    const long long b = first_block + blockIdx.x;
    const long long p = b / K2, k2 = b - p * K2;
    const size_t off = static_cast<size_t>(k2) * kChunk;
    const int n = So - off < static_cast<size_t>(kChunk) ? static_cast<int>(So - off) : kChunk;
    write_chunk<PAD, VEC>(in + static_cast<size_t>(p) * S, out + static_cast<size_t>(p) * So, off, n, h, w, Wo, pad,
                          Identity{});
}

bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

bool has_pad(const PlanePad* pad) { return pad && (pad->top | pad->bottom | pad->left | pad->right) != 0; }

// Launches kern over `blocks` CTAs in slices of at most kMaxBlocks, each told its first block.
template <class Launch>
void for_slices(long long blocks, Launch launch) {
    for (long long b0 = 0; b0 < blocks; b0 += kMaxBlocks) {
        launch(static_cast<unsigned>(blocks - b0 < kMaxBlocks ? blocks - b0 : kMaxBlocks), b0);
        count_launch();
    }
}

}  // namespace

size_t instance_norm_workspace_floats(int channels, size_t plane, int batch) {
    return 2 * static_cast<size_t>(channels) * batch * ceil_div_sz(plane, kChunk);
}

int instance_norm_forward(const float* in, float* out, int channels, int h, int w, const float* gamma,
                          const float* beta, float eps, int relu, const PlanePad* pad, float* workspace, int batch,
                          cudaStream_t s) {
    const bool padded = has_pad(pad);
    const PlanePad pd = padded ? *pad : PlanePad{0, 0, 0, 0, 0, 0.f};
    const size_t S = static_cast<size_t>(h) * w;
    const int Ho = h + pd.top + pd.bottom, Wo = w + pd.left + pd.right;
    const size_t So = static_cast<size_t>(Ho) * Wo;
    const long long planes = static_cast<long long>(batch) * channels;
    const long long K = static_cast<long long>(ceil_div_sz(S, kChunk)), K2 = static_cast<long long>(ceil_div_sz(So, kChunk));
    const int prof = prof_begin(s, PROF_INSTANCE_NORM, 0, 0, 4.0 * planes * (static_cast<double>(S) + So));
    const bool vin = S % 4 == 0 && aligned16(in);
    if (vin)
        for_slices(planes * K, [&](unsigned nb, long long b0) {
            instance_norm_stats_kernel<true><<<nb, kThreads, 0, s>>>(in, workspace, S, K, b0);
        });
    else
        for_slices(planes * K, [&](unsigned nb, long long b0) {
            instance_norm_stats_kernel<false><<<nb, kThreads, 0, s>>>(in, workspace, S, K, b0);
        });
    FCUDA_CHECK_LAUNCH();
    const bool vout = So % 4 == 0 && aligned16(out) && (padded || vin);
#define FCUDA_IN_APPLY(P, V)                                                                                          \
    for_slices(planes * K2, [&](unsigned nb, long long b0) {                                                          \
        instance_norm_apply_kernel<P, V><<<nb, kThreads, 0, s>>>(in, out, workspace, gamma, beta, eps, relu, channels, \
                                                                 h, w, S, K, Wo, So, K2, pd, b0);                     \
    })
    if (padded && vout) FCUDA_IN_APPLY(true, true);
    else if (padded) FCUDA_IN_APPLY(true, false);
    else if (vout) FCUDA_IN_APPLY(false, true);
    else FCUDA_IN_APPLY(false, false);
#undef FCUDA_IN_APPLY
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    return 0;
}

int padding_forward(const float* in, float* out, int channels, int h, int w, const PlanePad& pad, int batch,
                    cudaStream_t s) {
    const size_t S = static_cast<size_t>(h) * w;
    const int Wo = w + pad.left + pad.right;
    const size_t So = static_cast<size_t>(h + pad.top + pad.bottom) * Wo;
    const long long planes = static_cast<long long>(batch) * channels;
    const long long K2 = static_cast<long long>(ceil_div_sz(So, kChunk));
    const int prof = prof_begin(s, PROF_INSTANCE_NORM, 0, 0, 4.0 * planes * (static_cast<double>(S) + So));
    const bool padded = has_pad(&pad);
    const bool vout = So % 4 == 0 && aligned16(out) && (padded || aligned16(in));
#define FCUDA_PAD_LAUNCH(P, V)                                                                                        \
    for_slices(planes * K2, [&](unsigned nb, long long b0) {                                                          \
        padding_kernel<P, V><<<nb, kThreads, 0, s>>>(in, out, h, w, S, Wo, So, K2, pad, b0);                          \
    })
    if (padded && vout) FCUDA_PAD_LAUNCH(true, true);
    else if (padded) FCUDA_PAD_LAUNCH(true, false);
    else if (vout) FCUDA_PAD_LAUNCH(false, true);
    else FCUDA_PAD_LAUNCH(false, false);
#undef FCUDA_PAD_LAUNCH
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    return 0;
}

}  // namespace fcuda
