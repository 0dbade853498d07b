// Deconvolution (transposed convolution, ncnn's Deconvolution / DeconvolutionDepthWise) on top of the convolution paths.
//
// The contraction is rewritten as an ordinary stride-1 convolution so that it runs through fcuda_conv_* (tuned algorithm
// choice, halo kernel, BF16x3 / 3xTF32 / TF32, Winograd where it is chosen).  Output row Y = s*t + r of the
// deconvolution receives the taps ky = r + s*v only, with input row t - v; so all s_h*s_w output phases are the output
// channels of ONE convolution with kernel T = ceil(K/s), pads T-1 and the phase filters W'[(g, r_y, r_x, oc)][ic][u][v] =
// w[g*OCg + oc][ic][r_y + s_h*(T_h-1-u)][r_x + s_w*(T_w-1-v)] (0 past the kernel).  A scatter kernel then interleaves the
// phases into the cropped output, adding the bias once and applying the ReLU.  Stride 1 needs no phases: the flipped
// filter with dilation d and pads d*(K-1) - pad writes the output directly.  True depthwise layers have one input channel
// per filter, too little work for the tensor cores, and run as a CUDA-core gather.
//
// The scatter with stride r, no pads, no bias and no ReLU is ncnn's PixelShuffle (fcuda_pixel_shuffle_forward), and its
// ADD variant also adds a nearest-upsampled blob to each output: SRVGGNetCompact's tail, pixel_shuffle(conv) +
// nearest_upsample(x), as one read of each input and one write of the output.
#include "fcuda.h"

#include "common.cuh"
#include "deconv.cuh"
#include "resize.cuh"

#include <stdint.h>
#include <string.h>

#include <vector>

namespace fcuda {

constexpr int kDeconvThreads = 256;
constexpr int kDeconvMaxGridY = 65535;

constexpr int kScatterVec = 4;  // consecutive outputs of one row per thread

// One thread writes kScatterVec consecutive outputs of a row in every plane it visits: the row's phase ry, the columns'
// phases, source offsets and validity are worked out once per thread, so a plane costs the thread one 32-bit division
// (its group) and four independent loads before its stores.  Planes advance by gridDim.y with (n, oc) carried along,
// so no 64-bit division runs on the device.  ADD: the PixelShuffle tail's nearest-upsampled addend (deconv.cuh).
// VEC: OW % 4 == 0 and `out` 16-byte aligned, so the four outputs are one float4 store.
template <bool ADD, bool VEC>
__global__ void __launch_bounds__(kDeconvThreads)
deconv_scatter_kernel(const float* __restrict__ P, const float* __restrict__ bias, float* __restrict__ out,
                      DeconvScatterGeom g, int relu, long long planes, ScatterAddend a) {
    const int groups = (g.OW + kScatterVec - 1) / kScatterVec;  // per output row
    const int item = blockIdx.x * kDeconvThreads + threadIdx.x;
    if (item >= g.OH * groups) return;
    const int oy = item / groups, ox0 = (item - oy * groups) * kScatterVec;
    const int Y = oy + g.pad_top;
    const int ty = Y / g.stride_h, ry = Y - ty * g.stride_h;
    const int OCg = g.OC / g.group;
    const int OCp = g.OC * g.stride_h * g.stride_w;
    const size_t pc = static_cast<size_t>(g.Hc) * g.Wc;
    size_t off[kScatterVec];  // source offset of each output within its phase row: rx * OCg * pc + tx
    bool in[kScatterVec];     // a source element exists (0 in its place otherwise) and the output is inside the row
    bool col[kScatterVec];    // the output is inside the row
    int sx[kScatterVec];      // the addend's source column (the nearest Interp's map)
    {
        const int X = ox0 + g.pad_left;
        int tx = X / g.stride_w, rx = X - tx * g.stride_w;
#pragma unroll
        for (int k = 0; k < kScatterVec; ++k) {
            col[k] = VEC || ox0 + k < g.OW;
            in[k] = col[k] && ty < g.Hc && tx < g.Wc;
            off[k] = static_cast<size_t>(rx) * OCg * pc + tx;
            if constexpr (ADD) sx[k] = nearest_coord(ox0 + k, a.W, a.scale_w);
            if (++rx == g.stride_w) {
                rx = 0;
                ++tx;
            }
        }
    }
    const int sy = ADD ? nearest_coord(oy, a.H, a.scale_h) : 0;
    const size_t src_row = static_cast<size_t>(ty) * g.Wc;
    const size_t OHW = static_cast<size_t>(g.OH) * g.OW;
    const int step_n = gridDim.y / g.OC, step_oc = gridDim.y - step_n * g.OC;
    long long n = blockIdx.y / g.OC;
    int oc = blockIdx.y - static_cast<int>(n) * g.OC;
    for (long long plane = blockIdx.y; plane < planes; plane += gridDim.y) {  // plane = n * OC + oc
        const int grp = oc / OCg, ocg = oc - grp * OCg;
        const float* src = P + (static_cast<size_t>(n) * OCp + static_cast<size_t>(grp * g.stride_h + ry) * g.stride_w * OCg +
                                ocg) * pc + src_row;
        float v[kScatterVec];
#pragma unroll
        for (int k = 0; k < kScatterVec; ++k) v[k] = in[k] ? __ldg(src + off[k]) : 0.f;
        const float b = bias ? __ldg(bias + oc) : 0.f;
        const float* base = ADD ? a.base + (static_cast<size_t>(plane) * a.H + sy) * a.W : nullptr;
#pragma unroll
        for (int k = 0; k < kScatterVec; ++k) {
            if (bias) v[k] += b;
            if (relu) v[k] = v[k] > 0 ? v[k] : 0.f;  // the ReLU layer's comparison (layers.cu scale_relu_kernel)
            if constexpr (ADD) {
                if (col[k]) v[k] += __ldg(base + sx[k]);
            }
        }
        float* dst = out + static_cast<size_t>(plane) * OHW + static_cast<size_t>(oy) * g.OW + ox0;
        if constexpr (VEC) {
            *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int k = 0; k < kScatterVec; ++k)
                if (col[k]) dst[k] = v[k];
        }
        oc += step_oc;
        n += step_n;
        if (oc >= g.OC) {
            oc -= g.OC;
            ++n;
        }
    }
}

__global__ void __launch_bounds__(kDeconvThreads)
deconv_dw_gather_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                        float* __restrict__ out, DeconvDwGeom g, int relu, long long planes) {
    extern __shared__ float filt[];
    const int OHW = g.OH * g.OW, taps = g.KH * g.KW;
    const int idx = blockIdx.x * kDeconvThreads + threadIdx.x;
    const int oy = idx / g.OW, ox = idx - oy * g.OW;
    const int Y = oy + g.pad_top, X = ox + g.pad_left;
    // first tap of each direction: ky = Y mod s (stride > 1 implies dilation 1), then every s-th; with stride 1 every tap
    const int ky0 = Y % g.stride_h, kx0 = X % g.stride_w;
    for (long long plane = blockIdx.y; plane < planes; plane += gridDim.y) {  // plane = n * C + c
        const int c = static_cast<int>(plane % g.C);
        __syncthreads();
        for (int i = threadIdx.x; i < taps; i += kDeconvThreads) filt[i] = __ldg(w + static_cast<size_t>(c) * taps + i);
        __syncthreads();
        if (idx >= OHW) continue;
        const float* ip = in + static_cast<size_t>(plane) * g.H * g.W;
        float v = bias ? __ldg(bias + c) : 0.f;
        for (int ky = ky0; ky < g.KH; ky += g.stride_h) {
            const int ny = Y - ky * g.dil_h;
            if (ny < 0) break;  // rows only decrease from here
            const int iy = ny / g.stride_h;
            if (iy >= g.H) continue;
            for (int kx = kx0; kx < g.KW; kx += g.stride_w) {
                const int nx = X - kx * g.dil_w;
                if (nx < 0) break;
                const int ix = nx / g.stride_w;
                if (ix >= g.W) continue;
                v = fmaf(__ldg(ip + static_cast<size_t>(iy) * g.W + ix), filt[ky * g.KW + kx], v);
            }
        }
        if (relu) v = v > 0 ? v : 0.f;
        out[static_cast<size_t>(plane) * OHW + idx] = v;
    }
}

static dim3 plane_grid(int per_plane, long long planes) {
    return dim3(static_cast<unsigned>(ceil_div(per_plane, kDeconvThreads)),
                static_cast<unsigned>(planes < kDeconvMaxGridY ? planes : kDeconvMaxGridY));
}

int deconv_scatter(const float* P, const float* bias, float* out, const DeconvScatterGeom& g, int relu,
                   const ScatterAddend* add, int kind, int batch, cudaStream_t s) {
    const long long planes = static_cast<long long>(batch) * g.OC;
    const double out_n = static_cast<double>(planes) * g.OH * g.OW;
    const double p_n = static_cast<double>(batch) * g.OC * g.stride_h * g.stride_w * g.Hc * g.Wc;
    const double add_n = add ? static_cast<double>(planes) * add->H * add->W : 0.0;
    const int prof = prof_begin(s, kind, 0, 0, 4.0 * (out_n + p_n + add_n));
    const dim3 grid = plane_grid(g.OH * ceil_div(g.OW, kScatterVec), planes);
    const bool vec = g.OW % kScatterVec == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    const ScatterAddend a = add ? *add : ScatterAddend{};
    if (add && vec) deconv_scatter_kernel<true, true><<<grid, kDeconvThreads, 0, s>>>(P, bias, out, g, relu, planes, a);
    else if (add) deconv_scatter_kernel<true, false><<<grid, kDeconvThreads, 0, s>>>(P, bias, out, g, relu, planes, a);
    else if (vec) deconv_scatter_kernel<false, true><<<grid, kDeconvThreads, 0, s>>>(P, bias, out, g, relu, planes, a);
    else deconv_scatter_kernel<false, false><<<grid, kDeconvThreads, 0, s>>>(P, bias, out, g, relu, planes, a);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int deconv_depthwise(const float* in, const float* w, const float* bias, float* out, const DeconvDwGeom& g, int relu,
                     int batch, cudaStream_t s) {
    const long long planes = static_cast<long long>(batch) * g.C;
    const int smem = g.KH * g.KW * static_cast<int>(sizeof(float));
    if (smem > 48 * 1024) return -200;
    const double flops = 2.0 * planes * g.H * g.W * g.KH * g.KW;
    const int prof = prof_begin(s, PROF_DECONV, flops, 0,
                                4.0 * planes * (static_cast<double>(g.H) * g.W + static_cast<double>(g.OH) * g.OW));
    deconv_dw_gather_kernel<<<plane_grid(g.OH * g.OW, planes), kDeconvThreads, smem, s>>>(in, w, bias, out, g, relu, planes);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda

using namespace fcuda;

namespace {

enum DeconvPath { PATH_DEPTHWISE, PATH_DIRECT, PATH_SUBPIXEL };

struct DeconvPlan {
    int path = PATH_SUBPIXEL;
    FcudaConvParam eq{};
    int algo = -1;
    int dil_h = 1, dil_w = 1;  // of the equivalent convolution
    int Th = 0, Tw = 0;        // its kernel on the sub-pixel path
};

bool is_depthwise(const FcudaDeconvParam* p) {
    return p->group > 1 && p->group == p->input_channels && p->output_channels == p->input_channels;
}

int check_and_size(FcudaDeconvParam* p) {
    if (!p) return -100;
    if (p->output_channels <= 0 || p->input_channels <= 0 || p->input_h <= 0 || p->input_w <= 0 || p->kernel_h <= 0 ||
        p->kernel_w <= 0 || p->stride_h <= 0 || p->stride_w <= 0 || p->dilation_h <= 0 || p->dilation_w <= 0)
        return -100;
    if (p->pad_left < 0 || p->pad_right < 0 || p->pad_top < 0 || p->pad_bottom < 0 || p->output_pad_right < 0 ||
        p->output_pad_bottom < 0)
        return -200;
    if (p->activation != FCUDA_ACT_NONE && p->activation != FCUDA_ACT_RELU) return -200;
    if ((p->stride_h > 1 && p->dilation_h > 1) || (p->stride_w > 1 && p->dilation_w > 1)) return -200;
    if (p->group <= 0 || p->output_channels % p->group || p->input_channels % p->group) return -200;
    const long long hf = static_cast<long long>(p->input_h - 1) * p->stride_h +
                         static_cast<long long>(p->dilation_h) * (p->kernel_h - 1) + 1 + p->output_pad_bottom;
    const long long wf = static_cast<long long>(p->input_w - 1) * p->stride_w +
                         static_cast<long long>(p->dilation_w) * (p->kernel_w - 1) + 1 + p->output_pad_right;
    const long long oh = hf - p->pad_top - p->pad_bottom, ow = wf - p->pad_left - p->pad_right;
    if (oh <= 0 || ow <= 0 || oh * ow > 0x7fffffffLL) return -100;
    p->output_h = static_cast<int>(oh);
    p->output_w = static_cast<int>(ow);
    return 0;
}

int select_equivalent_algo(DeconvPlan& pl) {
    int rc;
    if (pl.dil_h > 1 || pl.dil_w > 1 || pl.eq.group > 1) {
        pl.algo = FCUDA_SGECONV;  // the only path that spaces taps or splits partial groups
    } else if ((rc = fcuda_conv_select_algo_tuned(&pl.eq, &pl.algo))) {
        return rc;
    }
    size_t a, b;
    return fcuda_conv_get_buffer_size(&pl.eq, pl.algo, 1, &a, &b);  // the convolution paths accept this geometry
}

int make_plan(const FcudaDeconvParam* in, DeconvPlan* out) {
    if (!in) return -100;
    FcudaDeconvParam p = *in;
    int rc = check_and_size(&p);
    if (rc) return rc;
    DeconvPlan pl;
    if (is_depthwise(&p)) {
        if (p.kernel_h * p.kernel_w * static_cast<long long>(sizeof(float)) > 48 * 1024) return -200;
        pl.path = PATH_DEPTHWISE;
        pl.algo = FCUDA_DEPTHWISE;
        *out = pl;
        return 0;
    }
    FcudaConvParam& e = pl.eq;
    e.input_channels = p.input_channels;
    e.input_h = p.input_h;
    e.input_w = p.input_w;
    e.stride_h = e.stride_w = 1;
    e.group = p.group;
    const int eh = p.dilation_h * (p.kernel_h - 1), ew = p.dilation_w * (p.kernel_w - 1);  // dilated kernel extents - 1
    const bool direct = p.stride_h == 1 && p.stride_w == 1 && p.pad_top <= eh && p.pad_bottom <= eh &&
                        p.pad_left <= ew && p.pad_right <= ew && p.output_pad_bottom <= p.pad_bottom &&
                        p.output_pad_right <= p.pad_right;
    if (direct) {
        pl.path = PATH_DIRECT;
        pl.dil_h = p.dilation_h;
        pl.dil_w = p.dilation_w;
        e.output_channels = p.output_channels;
        e.kernel_h = p.kernel_h;
        e.kernel_w = p.kernel_w;
        e.pad_top = eh - p.pad_top;
        e.pad_bottom = eh - p.pad_bottom + p.output_pad_bottom;
        e.pad_left = ew - p.pad_left;
        e.pad_right = ew - p.pad_right + p.output_pad_right;
        e.bias_term = static_cast<unsigned char>(p.bias_term != 0);
        e.activation = p.activation;
        e.output_h = p.output_h;
        e.output_w = p.output_w;
    } else {
        pl.path = PATH_SUBPIXEL;
        pl.dil_h = p.stride_h == 1 ? p.dilation_h : 1;
        pl.dil_w = p.stride_w == 1 ? p.dilation_w : 1;
        pl.Th = ceil_div(p.kernel_h, p.stride_h);
        pl.Tw = ceil_div(p.kernel_w, p.stride_w);
        const long long ocp = static_cast<long long>(p.output_channels) * p.stride_h * p.stride_w;
        if (ocp > 0x7fffffffLL) return -100;
        e.output_channels = static_cast<int>(ocp);
        e.kernel_h = pl.Th;
        e.kernel_w = pl.Tw;
        e.pad_top = e.pad_bottom = pl.dil_h * (pl.Th - 1);
        e.pad_left = e.pad_right = pl.dil_w * (pl.Tw - 1);
        e.bias_term = 0;
        e.activation = FCUDA_ACT_NONE;
        e.output_h = p.input_h + pl.dil_h * (pl.Th - 1);
        e.output_w = p.input_w + pl.dil_w * (pl.Tw - 1);
    }
    if ((rc = select_equivalent_algo(pl))) return rc;
    *out = pl;
    return 0;
}

// scratch of the equivalent convolution, rounded so that the phase planes after it start 256-byte aligned
int conv_scratch_floats(const DeconvPlan& pl, int batch, size_t* n) {
    size_t s = 0, k = 0;
    const int rc = fcuda_conv_get_buffer_size(&pl.eq, pl.algo, batch, &s, &k);
    *n = round_up_sz(s, 64);
    return rc;
}

size_t phase_floats(const DeconvPlan& pl, int batch) {
    if (pl.path != PATH_SUBPIXEL) return 0;
    return static_cast<size_t>(batch) * pl.eq.output_channels * pl.eq.output_h * pl.eq.output_w;
}

}  // namespace

extern "C" {

int fcuda_deconv_output_dim(FcudaDeconvParam* p) { return check_and_size(p); }

int fcuda_deconv_plan(const FcudaDeconvParam* p, FcudaConvParam* equivalent, int* conv_algo) {
    DeconvPlan pl;
    const int rc = make_plan(p, &pl);
    if (rc) return rc;
    if (equivalent) *equivalent = pl.eq;
    if (conv_algo) *conv_algo = pl.algo;
    return 0;
}

int fcuda_deconv_get_buffer_size(const FcudaDeconvParam* p, int batch, size_t* scratch_floats, size_t* packed_floats) {
    if (batch < 1) return -100;
    DeconvPlan pl;
    int rc = make_plan(p, &pl);
    if (rc) return rc;
    size_t scratch = 0, packed = 0;
    if (pl.path == PATH_DEPTHWISE) {
        packed = static_cast<size_t>(p->input_channels) * p->kernel_h * p->kernel_w;
    } else {
        if ((rc = conv_scratch_floats(pl, batch, &scratch))) return rc;
        scratch += phase_floats(pl, batch);
        size_t s1 = 0;
        if ((rc = fcuda_conv_get_buffer_size(&pl.eq, pl.algo, 1, &s1, &packed))) return rc;
    }
    if (scratch_floats) *scratch_floats = scratch;
    if (packed_floats) *packed_floats = packed;
    return 0;
}

int fcuda_deconv_init(const FcudaDeconvParam* p, float* packed, const float* raw, void* stream) {
    DeconvPlan pl;
    int rc = make_plan(p, &pl);
    if (rc) return rc;
    if (!packed || !raw) return -100;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int OC = p->output_channels, G = p->group, OCg = OC / G, ICg = p->input_channels / G;
    const int KH = p->kernel_h, KW = p->kernel_w;
    const size_t raw_n = static_cast<size_t>(OC) * ICg * KH * KW;
    // Init runs once per layer and precision mode: the filter is rearranged on the host
    std::vector<float> w(raw_n);
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, raw) == cudaSuccess &&
        (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) {
        FCUDA_CHECK(cudaStreamSynchronize(s));
        FCUDA_CHECK(cudaMemcpy(w.data(), raw, raw_n * sizeof(float), cudaMemcpyDeviceToHost));
    } else {
        cudaGetLastError();
        memcpy(w.data(), raw, raw_n * sizeof(float));
    }
    if (pl.path == PATH_DEPTHWISE) {
        FCUDA_CHECK(cudaMemcpyAsync(packed, w.data(), raw_n * sizeof(float), cudaMemcpyHostToDevice, s));
        FCUDA_CHECK(cudaStreamSynchronize(s));
        return 0;
    }
    std::vector<float> eqw;
    if (pl.path == PATH_DIRECT) {  // flipped filter
        eqw.resize(raw_n);
        for (size_t f = 0; f < static_cast<size_t>(OC) * ICg; ++f)
            for (int u = 0; u < KH; ++u)
                for (int v = 0; v < KW; ++v)
                    eqw[(f * KH + u) * KW + v] = w[(f * KH + (KH - 1 - u)) * KW + (KW - 1 - v)];
    } else {  // phase filters W'[(g, ry, rx, oc)][ic][u][v]
        const int SH = p->stride_h, SW = p->stride_w, TH = pl.Th, TW = pl.Tw;
        eqw.assign(static_cast<size_t>(pl.eq.output_channels) * ICg * TH * TW, 0.f);
        for (int g = 0; g < G; ++g)
            for (int ry = 0; ry < SH; ++ry)
                for (int rx = 0; rx < SW; ++rx)
                    for (int oc = 0; oc < OCg; ++oc) {
                        const size_t dst_oc = ((static_cast<size_t>(g) * SH + ry) * SW + rx) * OCg + oc;
                        const size_t src_oc = static_cast<size_t>(g) * OCg + oc;
                        for (int ic = 0; ic < ICg; ++ic)
                            for (int u = 0; u < TH; ++u) {
                                const int ky = ry + SH * (TH - 1 - u);
                                if (ky >= KH) continue;
                                for (int v = 0; v < TW; ++v) {
                                    const int kx = rx + SW * (TW - 1 - v);
                                    if (kx >= KW) continue;
                                    eqw[((dst_oc * ICg + ic) * TH + u) * TW + v] =
                                        w[((src_oc * ICg + ic) * KH + ky) * KW + kx];
                                }
                            }
                    }
    }
    return fcuda_conv_init(&pl.eq, pl.algo, packed, eqw.data(), stream);  // stages the host filter, synchronous
}

int fcuda_deconv_forward(const FcudaDeconvParam* p, float* output, const float* input, const float* packed,
                         float* scratch, const float* bias, int batch, void* stream) {
    if (batch < 1) return -100;
    DeconvPlan pl;
    int rc = make_plan(p, &pl);
    if (rc) return rc;
    if (!output || !input || !packed) return -100;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const float* b = p->bias_term ? bias : nullptr;
    if (p->bias_term && !bias) return -100;
    const int relu = p->activation == FCUDA_ACT_RELU;
    FcudaDeconvParam q = *p;
    check_and_size(&q);
    if (pl.path == PATH_DEPTHWISE) {
        DeconvDwGeom g;
        g.C = q.input_channels; g.H = q.input_h; g.W = q.input_w; g.KH = q.kernel_h; g.KW = q.kernel_w;
        g.stride_h = q.stride_h; g.stride_w = q.stride_w; g.dil_h = q.dilation_h; g.dil_w = q.dilation_w;
        g.pad_top = q.pad_top; g.pad_left = q.pad_left; g.OH = q.output_h; g.OW = q.output_w;
        return deconv_depthwise(input, packed, b, output, g, relu, batch, s);
    }
    size_t conv_scratch = 0;
    if ((rc = conv_scratch_floats(pl, batch, &conv_scratch))) return rc;
    if ((conv_scratch || pl.path == PATH_SUBPIXEL) && !scratch) return -100;
    FcudaConvOptions o{};
    o.dilation_h = pl.dil_h; o.dilation_w = pl.dil_w;
    if (pl.path == PATH_DIRECT)
        return fcuda_conv_forward_opts(&pl.eq, pl.algo, output, input, packed, scratch, b, &o, batch, stream);
    float* P = scratch + conv_scratch;
    if ((rc = fcuda_conv_forward_opts(&pl.eq, pl.algo, P, input, packed, scratch, nullptr, &o, batch, stream))) return rc;
    DeconvScatterGeom g;
    g.OC = q.output_channels; g.group = q.group; g.stride_h = q.stride_h; g.stride_w = q.stride_w;
    g.Hc = pl.eq.output_h; g.Wc = pl.eq.output_w; g.OH = q.output_h; g.OW = q.output_w;
    g.pad_top = q.pad_top; g.pad_left = q.pad_left;
    return deconv_scatter(P, b, output, g, relu, nullptr, PROF_DECONV, batch, s);
}

}  // extern "C"
