// Bandwidth-bound layer kernels: pooling, BN/Scale, eltwise add, ReLU, softmax, dropout, channel copies.
// Each replaces an inline CPU loop of the reference (citations at each kernel).  All are single-pass,
// coalesced along the innermost (W / flattened) dimension; grid-stride loops sized from the SM count.
#include "layers.cuh"
#include "common.cuh"

#include <float.h>

namespace fcuda {

static inline unsigned grid_for(size_t n, int block) {
    size_t blocks = ceil_div_sz(n, block);
    const size_t cap = static_cast<size_t>(sm_count()) * 32;
    if (blocks > cap) blocks = cap;
    if (blocks == 0) blocks = 1;
    return static_cast<unsigned>(blocks);
}

// PoolingLayer::Forward, /root/reference/src/layers/pooling_layer.h:38-91.  Window start subtracts BOTH pads
// of an axis (:56, :67) — reproduced as is; max pooling starts from -FLT_MAX (:53), average divides by the
// number of in-bounds elements (:84).
__global__ void __launch_bounds__(256)
pooling_kernel(const float* __restrict__ in, float* __restrict__ out, PoolGeom g, size_t total) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const int ox = static_cast<int>(idx % g.OW);
        size_t t = idx / g.OW;
        const int oy = static_cast<int>(t % g.OH);
        const size_t plane = t / g.OH;
        const float* ip = in + plane * g.H * g.W;
        const int ys = oy * g.stride_h - g.pad_top - g.pad_bottom;
        const int xs = ox * g.stride_w - g.pad_left - g.pad_right;
        const int y0 = max(ys, 0), y1 = min(ys + g.KH, g.H);
        const int x0 = max(xs, 0), x1 = min(xs + g.KW, g.W);
        if (g.type == 0) {
            float m = -FLT_MAX;
            for (int y = y0; y < y1; ++y)
                for (int x = x0; x < x1; ++x) m = fmaxf(m, __ldg(ip + static_cast<size_t>(y) * g.W + x));
            out[idx] = m;
        } else {
            float s = 0.f;
            int cnt = 0;
            for (int y = y0; y < y1; ++y)
                for (int x = x0; x < x1; ++x) { s += __ldg(ip + static_cast<size_t>(y) * g.W + x); ++cnt; }
            out[idx] = s / static_cast<float>(cnt);
        }
    }
}

// 3x3 / stride 2 / no padding (ResNet-50's pool1, ceil mode: the last window may be clipped): a warp marches down 16 output
// rows of a 32-column strip; per input row a lane loads one float2 (columns 2*ox, 2*ox+1) and takes column 2*ox+2 from the
// next lane by shuffle; every input row is loaded once per strip (the generic kernel above issues 9 scalar loads and ~100
// instructions of 64-bit index math per output).
__global__ void __launch_bounds__(128)
pool3x3s2_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int OH, int OW, int type, long long items,
                 int xstrips, int ystrips) {
    const long long item = static_cast<long long>(blockIdx.x) * 4 + (threadIdx.x >> 5);
    if (item >= items) return;
    const int lane = threadIdx.x & 31;
    const int xs = static_cast<int>(item % xstrips);
    const long long t = item / xstrips;
    const int ys = static_cast<int>(t % ystrips);
    const long long plane = t / ystrips;
    const float* ip = in + plane * H * W;
    float* op = out + plane * OH * OW;
    const int ox = xs * 32 + lane, ix = 2 * ox;
    const int oy0 = ys * 16, oy1 = min(oy0 + 16, OH);
    const bool c0 = ix < W, c1 = ix + 1 < W, c2 = ix + 2 < W;          // which of the window's three columns exist
    const float pad = type == 0 ? -FLT_MAX : 0.f;
    const int ncol = (c0 ? 1 : 0) + (c1 ? 1 : 0) + (c2 ? 1 : 0);
    // horizontal reduction of one input row over this lane's window (max or sum of the in-bounds columns)
    auto hrow = [&](int iy, float& r) {
        float a = pad, b = pad;
        if (iy < H && c0) {
            if (c1) { const float2 v = __ldg(reinterpret_cast<const float2*>(ip + static_cast<long long>(iy) * W + ix)); a = v.x; b = v.y; }
            else a = __ldg(ip + static_cast<long long>(iy) * W + ix);
        }
        float c = __shfl_down_sync(0xffffffffu, a, 1);                  // next lane's first column = my third
        if (lane == 31) c = (iy < H && c2) ? __ldg(ip + static_cast<long long>(iy) * W + ix + 2) : pad;
        if (!c2) c = pad;
        r = type == 0 ? fmaxf(fmaxf(a, b), c) : a + b + c;
    };
    float carry;  // horizontal result of the row shared by two consecutive windows (row 2*oy)
    hrow(2 * oy0, carry);
    for (int oy = oy0; oy < oy1; ++oy) {
        float r1, r2;
        hrow(2 * oy + 1, r1);
        hrow(2 * oy + 2, r2);
        const int nrow = min(2 * oy + 3, H) - 2 * oy;
        float v = type == 0 ? fmaxf(fmaxf(carry, r1), r2) : (carry + r1 + r2) / static_cast<float>(nrow * ncol);
        if (ox < OW) op[static_cast<long long>(oy) * OW + ox] = v;
        carry = r2;
    }
}

// 2x2 / stride 2 / no padding on planes whose width is a multiple of 4 (every VGG pool): a thread reads one float4 of
// two consecutive rows and writes two outputs, 32-bit index math only; the generic kernel above spends ~100
// instructions per output on 64-bit div/mod and runs at 40% of HBM.
__global__ void __launch_bounds__(256)
pool2x2_kernel(const float* __restrict__ in, float* __restrict__ out, int W, int OW, int pairs, unsigned long long m_pairs,
               int type, unsigned total) {
    const unsigned idx = blockIdx.x * 256u + threadIdx.x;
    if (idx >= total) return;
    const unsigned row = pairs == 1 ? idx : static_cast<unsigned>(__umul64hi(idx, m_pairs));  // plane*OH + oy
    const unsigned pr = idx - row * pairs;
    const float4* ip = reinterpret_cast<const float4*>(in + static_cast<size_t>(row) * 2 * W) + pr;
    const float4 a = __ldg(ip), b = __ldg(ip + (W >> 2));
    float2 o;
    if (type == 0) {
        o.x = fmaxf(fmaxf(a.x, a.y), fmaxf(b.x, b.y));
        o.y = fmaxf(fmaxf(a.z, a.w), fmaxf(b.z, b.w));
    } else {  // same summation order as the generic kernel: row by row, left to right
        o.x = (((a.x + a.y) + b.x) + b.y) / 4.f;
        o.y = (((a.z + a.w) + b.z) + b.w) / 4.f;
    }
    reinterpret_cast<float2*>(out + static_cast<size_t>(row) * OW)[pr] = o;
}

// Global average / max pooling (kernel == whole plane): one warp per plane, shuffle reduction.
__global__ void __launch_bounds__(256)
global_pool_kernel(const float* __restrict__ in, float* __restrict__ out, int HW, int type, size_t planes) {
    const size_t warp = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= planes) return;
    const float* ip = in + warp * HW;
    float acc = type == 0 ? -FLT_MAX : 0.f;
    for (int i = lane; i < HW; i += 32) {
        const float v = __ldg(ip + i);
        acc = type == 0 ? fmaxf(acc, v) : acc + v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float other = __shfl_xor_sync(0xffffffffu, acc, o);
        acc = type == 0 ? fmaxf(acc, other) : acc + other;
    }
    if (lane == 0) out[warp] = type == 0 ? acc : acc / static_cast<float>(HW);
}

// booster::batchnorm<has_bias, has_scale, has_relu>, avx/generic_kernels.cpp:237-279 and
// booster::scale<has_bias>, :203-233, as one per-channel affine kernel:  y = act((a*x + b) * s + t).
__global__ void __launch_bounds__(256)
channel_affine_kernel(const float* __restrict__ in, float* __restrict__ out, int channels, size_t hw,
                      const float* __restrict__ mul, const float* __restrict__ add, const float* __restrict__ mul2,
                      const float* __restrict__ add2, int relu, size_t total) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const int c = static_cast<int>((idx / hw) % channels);
        float v = in[idx];
        v = mul ? fmaf(__ldg(mul + c), v, add ? __ldg(add + c) : 0.f) : (add ? v + __ldg(add + c) : v);
        if (mul2) v *= __ldg(mul2 + c);
        if (add2) v += __ldg(add2 + c);
        if (relu) v = fmaxf(v, 0.f);
        out[idx] = v;
    }
}

// booster::add_relu<fuse_relu>, avx/generic_kernels.cpp:138-169.
__global__ void __launch_bounds__(256)
add_relu_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, size_t n, int relu) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t n4 = n >> 2;
    const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    if (vec) {
        for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
            const float4 x = reinterpret_cast<const float4*>(a)[i], y = reinterpret_cast<const float4*>(b)[i];
            float4 r = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
            if (relu) r = make_float4(fmaxf(r.x, 0.f), fmaxf(r.y, 0.f), fmaxf(r.z, 0.f), fmaxf(r.w, 0.f));
            reinterpret_cast<float4*>(out)[i] = r;
        }
        for (size_t i = (n4 << 2) + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
            const float r = a[i] + b[i];
            out[i] = relu ? fmaxf(r, 0.f) : r;
        }
    } else {
        for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
            const float r = a[i] + b[i];
            out[i] = relu ? fmaxf(r, 0.f) : r;
        }
    }
}

// Eltwise beyond the reference's SUM (eltwise_layer.h:57-66 rejects PROD / MAX / coefficients; semantics follow ncnn's
// Eltwise): op 0 = a*b, 1 = ca*a + cb*b, 2 = max(a, b); optional ReLU.
__global__ void __launch_bounds__(256)
eltwise_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, size_t n, int op,
               float ca, float cb, int relu) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float x = a[i], y = b[i];
        float r = op == 0 ? x * y : op == 1 ? fmaf(ca, x, cb * y) : fmaxf(x, y);
        out[i] = relu ? fmaxf(r, 0.f) : r;
    }
}

// ReluLayer::Forward (relu_layer.h:29-41) and DropoutLayer::Forward (dropout_layer.h:36-57): y = act(x * scale).
__global__ void __launch_bounds__(256)
scale_relu_kernel(const float* __restrict__ in, float* __restrict__ out, size_t n, float scale, int relu) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t n4 = n >> 2;
    const bool vec = ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const size_t nv = vec ? n4 : 0;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
        float4 x = reinterpret_cast<const float4*>(in)[i];
        if (scale != 1.f) x = make_float4(x.x * scale, x.y * scale, x.z * scale, x.w * scale);
        if (relu) x = make_float4(x.x > 0 ? x.x : 0.f, x.y > 0 ? x.y : 0.f, x.z > 0 ? x.z : 0.f, x.w > 0 ? x.w : 0.f);
        reinterpret_cast<float4*>(out)[i] = x;
    }
    for (size_t i = (nv << 2) + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float x = in[i];
        if (scale != 1.f) x *= scale;
        if (relu) x = x > 0 ? x : 0.f;
        out[i] = x;
    }
}

// ncnn's Clip (and Caffe's ReLU6 = Clip 0..6): y = min(max(x, lo), hi).  NaN becomes lo: fmaxf returns its non-NaN
// operand (ncnn's compare-and-assign passes NaN through).  In place (in == out) is allowed.
__global__ void __launch_bounds__(256)
clip_kernel(const float* in, float* out, size_t n, float lo, float hi) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const bool vec = ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const size_t nv = vec ? n >> 2 : 0;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
        const float4 x = reinterpret_cast<const float4*>(in)[i];
        reinterpret_cast<float4*>(out)[i] = make_float4(fminf(fmaxf(x.x, lo), hi), fminf(fmaxf(x.y, lo), hi),
                                                        fminf(fmaxf(x.z, lo), hi), fminf(fmaxf(x.w, lo), hi));
    }
    for (size_t i = (nv << 2) + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = fminf(fmaxf(in[i], lo), hi);
}

// ncnn's PReLU: y = x < 0 ? x * slope[c] : x over (batch, channels, plane); one slope per channel, or slope[0] for all
// (shared).  VEC: plane % 4 == 0 and 16-byte aligned tensors, so a float4 never straddles two channels.  In place allowed.
template <bool VEC>
__global__ void __launch_bounds__(256)
prelu_kernel(const float* in, float* out, const float* __restrict__ slope, int channels, size_t plane, int shared,
             size_t n) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t items = VEC ? n >> 2 : n;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < items; i += stride) {
        const size_t e = VEC ? i << 2 : i;
        const float a = __ldg(slope + (shared ? 0 : static_cast<int>((e / plane) % channels)));
        if (VEC) {
            float4 x = reinterpret_cast<const float4*>(in)[i];
            x = make_float4(x.x < 0.f ? x.x * a : x.x, x.y < 0.f ? x.y * a : x.y, x.z < 0.f ? x.z * a : x.z,
                            x.w < 0.f ? x.w * a : x.w);
            reinterpret_cast<float4*>(out)[i] = x;
        } else {
            const float x = in[i];
            out[i] = x < 0.f ? x * a : x;
        }
    }
}

// SoftmaxLayer::Forward, softmax_layer.h:32-55: max-subtracted softmax over the whole blob of one image.
// One block per image.
__global__ void __launch_bounds__(256)
softmax_kernel(const float* __restrict__ in, float* __restrict__ out, size_t n) {
    __shared__ float red[8];
    __shared__ float bcast;
    const float* ip = in + static_cast<size_t>(blockIdx.x) * n;
    float* op = out + static_cast<size_t>(blockIdx.x) * n;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float m = -FLT_MAX;
    for (size_t i = threadIdx.x; i < n; i += 256) m = fmaxf(m, ip[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) red[warp] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float r = red[0];
        for (int i = 1; i < 8; ++i) r = fmaxf(r, red[i]);
        bcast = r;
    }
    __syncthreads();
    m = bcast;
    float s = 0.f;
    for (size_t i = threadIdx.x; i < n; i += 256) {
        const float e = expf(ip[i] - m);
        op[i] = e;
        s += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __syncthreads();
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float r = 0.f;
        for (int i = 0; i < 8; ++i) r += red[i];
        bcast = r;
    }
    __syncthreads();
    s = bcast;
    for (size_t i = threadIdx.x; i < n; i += 256) op[i] = op[i] / s;
}

// ConcatLayer::Forward (concat_layer.h:37-47) / SplitLayer::Forward (split_layer.h:43-53) per image.
__global__ void __launch_bounds__(256)
copy_channels_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t per_image, size_t dst_image,
                     size_t dst_offset, size_t total) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const size_t n = idx / per_image, r = idx - n * per_image;
        dst[n * dst_image + dst_offset + r] = src[idx];
    }
}

__global__ void __launch_bounds__(256)
fill_rows_kernel(float* __restrict__ out, const float* __restrict__ row, int row_len, size_t total) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride)
        out[idx] = row ? __ldg(row + idx % row_len) : 0.f;
}

// out[r][j] = act(bias[j] + part[0][r][j] + part[1][r][j] + ...): the k-split partial planes of the InnerProduct GEMM
// summed in a fixed order (deterministic, unlike atomics), bias and ReLU fused
__global__ void __launch_bounds__(256)
fc_reduce_kernel(float* __restrict__ out, const float* __restrict__ part, const float* __restrict__ bias, int splits,
                 size_t plane, int row_len, int relu) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < plane; idx += stride) {
        float v = bias ? __ldg(bias + idx % row_len) : 0.f;
        for (int s = 0; s < splits; ++s) v += __ldg(part + static_cast<size_t>(s) * plane + idx);
        out[idx] = relu ? fmaxf(v, 0.f) : v;
    }
}

// ------------------------------------------------------------------------------------------------
int pooling_forward(const float* in, float* out, const PoolGeom& g, int channels, int batch, cudaStream_t s) {
    const size_t planes = static_cast<size_t>(batch) * channels;
    const int prof = prof_begin(s, PROF_POOL, 0, 0, 4.0 * planes * (static_cast<double>(g.H) * g.W + static_cast<double>(g.OH) * g.OW));
    const uintptr_t ia = reinterpret_cast<uintptr_t>(in), oa = reinterpret_cast<uintptr_t>(out);
    if (g.OH == 1 && g.OW == 1 && g.KH >= g.H && g.KW >= g.W && g.pad_top + g.pad_bottom == 0 &&
        g.pad_left + g.pad_right == 0) {
        global_pool_kernel<<<static_cast<unsigned>(ceil_div_sz(planes * 32, 256)), 256, 0, s>>>(in, out, g.H * g.W,
                                                                                              g.type, planes);
    } else if (g.KH == 2 && g.KW == 2 && g.stride_h == 2 && g.stride_w == 2 && g.pad_top + g.pad_bottom == 0 &&
               g.pad_left + g.pad_right == 0 && g.W % 4 == 0 && g.H % 2 == 0 && g.OW == g.W / 2 && g.OH == g.H / 2 &&
               planes * g.OH * (g.OW / 2) < (1ull << 31) &&
               (ia & 15) == 0 && (oa & 7) == 0) {  // float4 loads, float2 stores: a C ABI caller may pass any float*
        const int pairs = g.OW / 2;
        const unsigned total = static_cast<unsigned>(planes * g.OH * pairs);
        const unsigned long long m = pairs > 1 ? ~0ull / static_cast<unsigned long long>(pairs) + 1ull : 0ull;
        pool2x2_kernel<<<(total + 255) / 256, 256, 0, s>>>(in, out, g.W, g.OW, pairs, m, g.type, total);
    } else if (g.KH == 3 && g.KW == 3 && g.stride_h == 2 && g.stride_w == 2 && g.pad_top + g.pad_bottom == 0 &&
               g.pad_left + g.pad_right == 0 && g.W % 2 == 0 && g.OW >= 24 && 2 * (g.OW - 1) < g.W && 2 * (g.OH - 1) < g.H &&
               (ia & 7) == 0) {  // float2 loads: the input 8-byte aligned
        const int xstrips = (g.OW + 31) / 32, ystrips = (g.OH + 15) / 16;
        const long long items = static_cast<long long>(planes) * xstrips * ystrips;
        pool3x3s2_kernel<<<static_cast<unsigned>((items + 3) / 4), 128, 0, s>>>(in, out, g.H, g.W, g.OH, g.OW, g.type, items,
                                                                              xstrips, ystrips);
    } else {
        const size_t total = planes * g.OH * g.OW;
        pooling_kernel<<<grid_for(total, 256), 256, 0, s>>>(in, out, g, total);
    }
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int channel_affine(const float* in, float* out, int channels, size_t hw, const float* mul, const float* add,
                   const float* mul2, const float* add2, int relu, int batch, cudaStream_t s) {
    const size_t total = static_cast<size_t>(batch) * channels * hw;
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, 8.0 * total);
    channel_affine_kernel<<<grid_for(total, 256), 256, 0, s>>>(in, out, channels, hw, mul, add, mul2, add2, relu, total);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int add_relu(const float* a, const float* b, float* out, size_t n, int relu, cudaStream_t s) {
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, 12.0 * n);
    add_relu_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, s>>>(a, b, out, n, relu);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int eltwise(const float* a, const float* b, float* out, size_t n, int op, float ca, float cb, int relu, cudaStream_t s) {
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, 12.0 * n);
    eltwise_kernel<<<grid_for(n, 256), 256, 0, s>>>(a, b, out, n, op, ca, cb, relu);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int scale_relu(const float* in, float* out, size_t n, float scale, int relu, cudaStream_t s) {
    scale_relu_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, s>>>(in, out, n, scale, relu);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int clip(const float* in, float* out, size_t n, float lo, float hi, cudaStream_t s) {
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, 8.0 * n);
    clip_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, s>>>(in, out, n, lo, hi);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int prelu(const float* in, float* out, const float* slope, int channels, size_t plane, int shared, int batch,
          cudaStream_t s) {
    const size_t n = static_cast<size_t>(batch) * channels * plane;
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, 8.0 * n + 4.0 * (shared ? 1 : channels));
    const bool vec = plane % 4 == 0 && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    if (vec) prelu_kernel<true><<<grid_for(n / 4 + 1, 256), 256, 0, s>>>(in, out, slope, channels, plane, shared, n);
    else prelu_kernel<false><<<grid_for(n, 256), 256, 0, s>>>(in, out, slope, channels, plane, shared, n);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int softmax_forward(const float* in, float* out, size_t n_per_image, int batch, cudaStream_t s) {
    softmax_kernel<<<batch, 256, 0, s>>>(in, out, n_per_image);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int copy_channels(const float* src, float* dst, size_t per_image, size_t dst_image, size_t dst_offset, int batch,
                  cudaStream_t s) {
    const size_t total = per_image * batch;
    copy_channels_kernel<<<grid_for(total, 256), 256, 0, s>>>(src, dst, per_image, dst_image, dst_offset, total);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int fc_reduce(float* out, const float* part, const float* bias, int splits, int row_len, int rows, int relu,
              cudaStream_t s) {
    const size_t plane = static_cast<size_t>(row_len) * rows;
    fc_reduce_kernel<<<grid_for(plane, 256), 256, 0, s>>>(out, part, bias, splits, plane, row_len, relu);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int fill_rows(float* out, const float* row, int row_len, int rows, cudaStream_t s) {
    const size_t total = static_cast<size_t>(row_len) * rows;
    fill_rows_kernel<<<grid_for(total, 256), 256, 0, s>>>(out, row, row_len, total);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
