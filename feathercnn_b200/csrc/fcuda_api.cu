// extern "C" surface of libfcuda.so (include/fcuda.h): algorithm selection, workspace planning and the
// per-layer dispatch that stands where booster::ConvBooster's function table stood
// (/root/reference/src/booster/avx/booster.cpp:283-355).
#include "fcuda.h"

#include "common.cuh"
#include "conv_direct.cuh"
#include "conv_igemm.cuh"
#include "depthwise.cuh"
#include "layers.cuh"
#include "pack.cuh"
#include "preprocess.cuh"
#include "tensor_gemm.cuh"
#include "winograd.cuh"

#include <math.h>
#include <stdlib.h>
#include <string.h>

using namespace fcuda;

namespace {

int env_precision() {
    const char* e = getenv("FCUDA_PRECISION");
    if (e && (!strcmp(e, "tf32") || !strcmp(e, "TF32") || !strcmp(e, "1"))) return FCUDA_PRECISION_TF32;
    if (e && (!strcmp(e, "tf32x3") || !strcmp(e, "3xtf32") || !strcmp(e, "0"))) return FCUDA_PRECISION_TF32X3;
    return FCUDA_PRECISION_FP32_SPLIT;
}
size_t env_chunk() {
    const char* e = getenv("FCUDA_L2_CHUNK_MB");
    if (e) return static_cast<size_t>(atof(e) * 1024.0 * 1024.0);
    // Default: effectively one chunk per layer (the Winograd / im2col intermediates of a layer exceed the L2 either way,
    // so smaller chunks only add launches and tail effects).  The bound keeps the scratch pool finite for very large
    // batches.
    return static_cast<size_t>(8) << 30;
}

int g_precision = env_precision();
size_t g_l2_chunk = env_chunk();

inline int planes() { return g_precision == FCUDA_PRECISION_TF32 ? 1 : 2; }
// operand format of the implicit GEMM (IgemmProblem::planes): 3 = BF16x3 in the default fp32-split mode
inline int igemm_planes() { return g_precision == FCUDA_PRECISION_FP32_SPLIT ? 3 : planes(); }
inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

struct ConvPlan {
    int algo = -1;
    int np = 1;  // operand planes (1 = TF32, 2 = 3xTF32)
    // Winograd
    int tile = 0, TT = 0;
    WinoGeom wg{};
    int total_tile_rows = 0, rows_per_chunk = 0;
    size_t Tc_max = 0;
    // im2col / direct
    PackGeom pg{};
    long long total_pixels = 0;
    int pixels_per_chunk = 0;
    bool im2col_tc = false;  // false => fall back to the CUDA-core direct kernel
    // depthwise
    DwGeom dg{};
    size_t scratch_floats = 0, packed_floats = 0;
};

PackGeom pack_geom(const FcudaConvParam* p) {
    PackGeom g;
    g.IC = p->input_channels; g.H = p->input_h; g.W = p->input_w;
    g.KH = p->kernel_h; g.KW = p->kernel_w; g.OH = p->output_h; g.OW = p->output_w;
    g.stride_h = p->stride_h; g.stride_w = p->stride_w; g.pad_top = p->pad_top; g.pad_left = p->pad_left;
    g.K = p->input_channels * p->kernel_h * p->kernel_w;
    g.Kp = (g.K + 3) & ~3;
    return g;
}

int make_plan(const FcudaConvParam* p, int algo, int batch, ConvPlan* plan) {
    if (!p || batch < 1) return -100;
    if (p->output_channels <= 0 || p->input_channels <= 0 || p->input_h <= 0 || p->input_w <= 0 ||
        p->kernel_h <= 0 || p->kernel_w <= 0 || p->stride_h <= 0 || p->stride_w <= 0 || p->output_h <= 0 ||
        p->output_w <= 0)
        return -100;
    ConvPlan& pl = *plan;
    pl.algo = algo;
    pl.np = planes();
    const int IC = p->input_channels, OC = p->output_channels;
    switch (algo) {
        case FCUDA_WINOGRADF63:
        case FCUDA_WINOGRADF23: {
            if (p->group != 1 || p->kernel_h != 3 || p->kernel_w != 3 || p->stride_h != 1 || p->stride_w != 1) return -1;
            if (IC % 4 != 0) return -1;  // TMA needs 16-byte rows (the reference's rule is IC%4 && OC%4 too)
            pl.tile = algo == FCUDA_WINOGRADF63 ? 8 : 4;
            pl.TT = pl.tile * pl.tile;
            const int ot = pl.tile - 2;
            WinoGeom& g = pl.wg;
            g.C_in = IC; g.C_out = OC; g.H = p->input_h; g.W = p->input_w; g.OH = p->output_h; g.OW = p->output_w;
            g.pad_top = p->pad_top; g.pad_left = p->pad_left;
            g.tilesX = ceil_div(g.OW, ot);  // == (Wp + 3) / 6 for F(6,3), winograd_kernels_F63.cpp:2320
            g.tilesY = ceil_div(g.OH, ot);
            pl.total_tile_rows = batch * g.tilesY;
            // V is stored once as plain fp32 (the TensorGEMM splits it in-kernel), M once
            const size_t bytes_per_row = static_cast<size_t>(g.tilesX) * pl.TT * (static_cast<size_t>(IC) + OC) * 4;
            const size_t u_bytes = static_cast<size_t>(pl.np) * pl.TT * IC * OC * 4;
            size_t budget = g_l2_chunk;
            if (budget && budget < 2 * u_bytes) budget = 2 * u_bytes;  // do not re-stream U more than the data it multiplies
            long long rows = budget ? static_cast<long long>(budget / bytes_per_row) : pl.total_tile_rows;
            if (rows < 1) rows = 1;
            if (rows > pl.total_tile_rows) rows = pl.total_tile_rows;
            const int nchunks = ceil_div(pl.total_tile_rows, static_cast<int>(rows));
            pl.rows_per_chunk = ceil_div(pl.total_tile_rows, nchunks);
            pl.Tc_max = static_cast<size_t>(pl.rows_per_chunk) * g.tilesX;
            if (pl.Tc_max > 0x7fffffffULL / 64) return -100;
            pl.scratch_floats = pl.TT * pl.Tc_max * (static_cast<size_t>(IC) + OC);
            pl.packed_floats = static_cast<size_t>(pl.np) * pl.TT * IC * OC;
            return 0;
        }
        case FCUDA_IM2COL:
        case FCUDA_NAIVE: {
            if (p->group != 1) return -1;
            pl.pg = pack_geom(p);
            pl.total_pixels = static_cast<long long>(batch) * p->output_h * p->output_w;
            if (algo == FCUDA_NAIVE) {
                pl.scratch_floats = 0;
                pl.packed_floats = static_cast<size_t>(OC) * pl.pg.K;
                return 0;
            }
            pl.im2col_tc = true;
            const size_t bytes_per_pixel = static_cast<size_t>(pl.pg.Kp) * 4;
            long long pix = g_l2_chunk ? static_cast<long long>(g_l2_chunk / bytes_per_pixel) : pl.total_pixels;
            pix = pix / 128 * 128;
            if (pix < 128) pix = 128;
            if (pix > pl.total_pixels) pix = pl.total_pixels;
            if (pix > 0x7fffff00LL) pix = 0x7fffff00LL;
            const long long nchunks = (pl.total_pixels + pix - 1) / pix;
            pix = ((pl.total_pixels + nchunks - 1) / nchunks + 127) / 128 * 128;
            pl.pixels_per_chunk = static_cast<int>(pix);
            pl.scratch_floats = static_cast<size_t>(pix) * pl.pg.Kp;
            pl.packed_floats = static_cast<size_t>(pl.np) * OC * pl.pg.Kp;
            return 0;
        }
        case FCUDA_SGECONV: {
            // implicit GEMM straight from NCHW: any kernel / stride / padding / dilation; group > 1 (an extension: the
            // reference returns -1 for partial groups, avx/booster.cpp:304-308) runs one launch per group on channel
            // slices, with input_channels / output_channels the TOTAL channel counts and weights (OC, IC/group, KH, KW)
            const int G = p->group > 0 ? p->group : 1;
            if (IC % G != 0 || OC % G != 0) return -1;
            if (!conv_igemm_supported(IC / G, p->kernel_h, p->kernel_w)) return -1;
            pl.pg = pack_geom(p);
            pl.scratch_floats = 0;
            pl.packed_floats = static_cast<size_t>(G) * conv_igemm_packed_floats(OC / G, IC / G, p->kernel_h * p->kernel_w, pl.np);
            return 0;
        }
        case FCUDA_DEPTHWISE: {
            if (p->group != IC || OC != IC) return -1;  // channel multiplier > 1: use FCUDA_SGECONV (grouped)
            DwGeom& g = pl.dg;
            g.C = IC; g.H = p->input_h; g.W = p->input_w; g.KH = p->kernel_h; g.KW = p->kernel_w;
            g.OH = p->output_h; g.OW = p->output_w; g.stride_h = p->stride_h; g.stride_w = p->stride_w;
            g.pad_top = p->pad_top; g.pad_left = p->pad_left;
            pl.scratch_floats = 0;
            pl.packed_floats = static_cast<size_t>(IC) * p->kernel_h * p->kernel_w;
            return 0;
        }
        default:
            // WINOGRADF63FUSED: unselected in the reference's AVX dispatcher and crashing as wired
            // (avx/booster.cpp:258, 291-292); "This algo is not supported" => -1 (booster.cpp:349-353).
            return -1;
    }
}

// Stage a possibly-host pointer on the device.  Returns the device pointer to use and, when a temporary
// was allocated, stores it in *tmp (caller frees after the consuming kernels are enqueued + synchronised).
int stage_to_device(const float* src, size_t n, const float** dev, float** tmp, cudaStream_t s) {
    *tmp = nullptr;
    cudaPointerAttributes attr;
    cudaError_t e = cudaPointerGetAttributes(&attr, src);
    if (e == cudaSuccess && (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) {
        *dev = src;
        return 0;
    }
    cudaGetLastError();
    FCUDA_CHECK(cudaMalloc(tmp, n * sizeof(float)));
    FCUDA_CHECK(cudaMemcpyAsync(*tmp, src, n * sizeof(float), cudaMemcpyHostToDevice, s));
    *dev = *tmp;
    return 0;
}

}  // namespace

extern "C" {

int fcuda_set_precision(int precision) {
    if (precision != FCUDA_PRECISION_TF32X3 && precision != FCUDA_PRECISION_TF32 && precision != FCUDA_PRECISION_FP32_SPLIT)
        return -200;
    g_precision = precision;
    return 0;
}
int fcuda_get_precision(void) { return g_precision; }
int fcuda_set_l2_chunk_bytes(size_t bytes) { g_l2_chunk = bytes; return 0; }
size_t fcuda_get_l2_chunk_bytes(void) { return g_l2_chunk; }

int fcuda_conv_assign_output_dim(FcudaConvParam* p) {
    if (!p) return -100;
    if (p->group == 0) p->group = 1;
    if (p->stride_h == 0) p->stride_h = 1;
    if (p->stride_w == 0) p->stride_w = 1;
    p->output_h = (p->input_h + p->pad_top + p->pad_bottom - p->kernel_h) / p->stride_h + 1;
    p->output_w = (p->input_w + p->pad_left + p->pad_right - p->kernel_w) / p->stride_w + 1;
    if (p->group == p->input_channels) p->output_channels = p->input_channels;
    return 0;
}

int fcuda_conv_select_algo(const FcudaConvParam* p, int* algo) {
    if (!p || !algo) return -100;
    if (p->group == p->input_channels) {
        *algo = FCUDA_DEPTHWISE;
    } else if (p->group == 1 && p->kernel_h == 3 && p->kernel_w == 3 && p->stride_h == 1 && p->stride_w == 1 &&
               p->input_h > 8 && p->input_w > 8 && p->output_channels % 4 == 0 && p->input_channels % 4 == 0) {
        *algo = FCUDA_WINOGRADF63;
    } else if (p->group == 1) {
        *algo = FCUDA_IM2COL;
    } else {
        *algo = -1;
        return -1;  // partial group conv, avx/booster.cpp:304-308
    }
    return 0;
}

int fcuda_conv_select_algo_tuned(const FcudaConvParam* p, int* algo) {
    if (!p || !algo) return -100;
    const int IC = p->input_channels, OC = p->output_channels;
    if (p->group > 1) {
        // true depthwise (one filter per channel) -> the stencil kernels; partial groups and channel-multiplier
        // depthwise (rejected by the reference, avx/booster.cpp:304-308) -> grouped implicit GEMM
        if (p->group == IC && OC == IC) { *algo = FCUDA_DEPTHWISE; return 0; }
        if (IC % p->group == 0 && OC % p->group == 0 && conv_igemm_supported(IC / p->group, p->kernel_h, p->kernel_w)) {
            *algo = FCUDA_SGECONV;
            return 0;
        }
        *algo = -1;
        return -1;
    }
    int rc;
    if (IC == 1) {
        // group == 1 with ONE input channel (grayscale / LeNet conv1) is an ordinary convolution; the reference's
        // `group == input_channels` test would turn it into a 1-output depthwise (avx/booster.cpp:285)
        *algo = FCUDA_IM2COL;
        rc = 0;
    } else {
        rc = fcuda_conv_select_algo(p, algo);
    }
    if (rc != 0 || *algo == FCUDA_DEPTHWISE) return rc;
    if (*algo == FCUDA_WINOGRADF63) {
        // non-fused Winograd moves 64/36 x (2*in + out) through HBM; below ~128 channels on large images that traffic
        // outweighs its 4.5x MMA saving and the single-kernel implicit GEMM wins
        if (IC <= 128 && OC <= 128 && p->output_w >= 28) *algo = FCUDA_SGECONV;
    } else if (*algo == FCUDA_IM2COL) {
        // everything the reference sends to im2col + SGEMM (1x1, strided, 7x7, IC = 3, small images): gather the
        // patches inside the GEMM instead of materialising them
        if (conv_igemm_supported(IC, p->kernel_h, p->kernel_w)) *algo = FCUDA_SGECONV;
    }
    return 0;
}

int fcuda_conv_get_buffer_size(const FcudaConvParam* p, int algo, int batch, size_t* scratch_floats,
                               size_t* packed_kernel_floats) {
    ConvPlan pl;
    const int rc = make_plan(p, algo, batch, &pl);
    if (rc) return rc;
    if (scratch_floats) *scratch_floats = pl.scratch_floats;
    if (packed_kernel_floats) *packed_kernel_floats = pl.packed_floats;
    return 0;
}

int fcuda_conv_init(const FcudaConvParam* p, int algo, float* packed, const float* raw, void* stream) {
    ConvPlan pl;
    int rc = make_plan(p, algo, 1, &pl);
    if (rc) return rc;
    if (!packed || !raw) return -100;
    cudaStream_t s = as_stream(stream);
    const int IC = p->input_channels, OC = p->output_channels;
    const size_t raw_n = algo == FCUDA_DEPTHWISE ? static_cast<size_t>(IC) * p->kernel_h * p->kernel_w
                                                 : static_cast<size_t>(OC) * (IC / (p->group > 0 ? p->group : 1)) *
                                                       p->kernel_h * p->kernel_w;
    const float* d_raw;
    float* tmp;
    if ((rc = stage_to_device(raw, raw_n, &d_raw, &tmp, s))) return rc;
    switch (algo) {
        case FCUDA_WINOGRADF63:
        case FCUDA_WINOGRADF23: {
            const size_t plane = static_cast<size_t>(pl.TT) * IC * OC;
            rc = wino_filter_transform(pl.tile, d_raw, packed, pl.np == 2 ? packed + plane : nullptr, OC, IC, s);
            break;
        }
        case FCUDA_IM2COL: {
            const size_t plane = static_cast<size_t>(OC) * pl.pg.Kp;
            rc = pack_weights(d_raw, packed, pl.np == 2 ? packed + plane : nullptr, OC, pl.pg.K, pl.pg.Kp, s);
            break;
        }
        case FCUDA_SGECONV: {
            const int taps = p->kernel_h * p->kernel_w;
            const int G = p->group > 0 ? p->group : 1;
            const int ICg = IC / G, OCg = OC / G;
            const size_t plane = conv_igemm_packed_floats(OCg, ICg, taps, 1);
            const size_t group_stride = conv_igemm_packed_floats(OCg, ICg, taps, pl.np);  // (the BF16x3 planes are pre-tiled and padded)
            for (int g = 0; g < G && rc == 0; ++g) {  // per group: [hi plane][lo plane] of Wp[OCg][Kf]
                float* dst = packed + static_cast<size_t>(g) * group_stride;
                rc = conv_igemm_pack_weights(d_raw + static_cast<size_t>(g) * OCg * ICg * taps, dst,
                                             pl.np == 2 ? dst + plane : nullptr, OCg, ICg, taps, s, igemm_planes() == 3);
            }
            break;
        }
        case FCUDA_NAIVE:
        case FCUDA_DEPTHWISE:
            if (cudaMemcpyAsync(packed, d_raw, raw_n * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
                rc = FCUDA_ERR_CUDA;
            break;
        default:
            rc = -1;
    }
    if (tmp) {
        cudaStreamSynchronize(s);
        cudaFree(tmp);
    }
    return rc;
}

static int conv_forward_impl(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                             float* scratch, const float* bias, const float* residual, int relu_after_add, int batch,
                             void* stream, int dil_h = 1, int dil_w = 1, int pool = 0);

int fcuda_conv_forward_ext(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                           float* scratch, const float* bias, const float* residual, int relu_after_add, int dilation_h,
                           int dilation_w, int batch, void* stream) {
    if (!p || dilation_h < 1 || dilation_w < 1) return -100;
    if ((dilation_h > 1 || dilation_w > 1) && algo != FCUDA_SGECONV) return -200;  // only the implicit GEMM spaces its taps
    if (residual && !(algo == FCUDA_SGECONV && p->activation == FCUDA_ACT_NONE)) {
        if (dilation_h > 1 || dilation_w > 1) return -200;
        return fcuda_conv_forward_residual(p, algo, output, input, packed, scratch, bias, residual, relu_after_add, batch, stream);
    }
    return conv_forward_impl(p, algo, output, input, packed, scratch, bias, residual, relu_after_add, batch, stream,
                             dilation_h, dilation_w);
}

int fcuda_conv_forward(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                       float* scratch, const float* bias, int batch, void* stream) {
    return conv_forward_impl(p, algo, output, input, packed, scratch, bias, nullptr, 0, batch, stream);
}

int fcuda_conv_forward_residual(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                                float* scratch, const float* bias, const float* residual, int relu_after_add, int batch,
                                void* stream) {
    if (!p || !residual) return -100;
    if (algo == FCUDA_SGECONV && p->activation == FCUDA_ACT_NONE)  // fused into the implicit-GEMM epilogue
        return conv_forward_impl(p, algo, output, input, packed, scratch, bias, residual, relu_after_add, batch, stream);
    // every other algorithm: the convolution, then the reference's add_relu in place
    int rc = conv_forward_impl(p, algo, output, input, packed, scratch, bias, nullptr, 0, batch, stream);
    if (rc) return rc;
    const size_t n = static_cast<size_t>(batch) * p->output_channels * p->output_h * p->output_w;
    return add_relu(output, residual, output, n, relu_after_add, as_stream(stream));
}

static int conv_forward_impl(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                             float* scratch, const float* bias, const float* residual, int relu_after_add, int batch,
                             void* stream, int dil_h, int dil_w, int pool) {
    ConvPlan pl;
    int rc = make_plan(p, algo, batch, &pl);
    if (rc) return rc;
    if (!output || !input || !packed) return -100;
    if (pl.scratch_floats && !scratch) return -100;
    cudaStream_t s = as_stream(stream);
    const int IC = p->input_channels, OC = p->output_channels;
    const float* b = p->bias_term ? bias : nullptr;
    const int relu = p->activation == FCUDA_ACT_RELU;
    switch (algo) {
        case FCUDA_WINOGRADF63:
        case FCUDA_WINOGRADF23: {
            const size_t v_plane = static_cast<size_t>(pl.TT) * pl.Tc_max * IC;
            const size_t u_plane = static_cast<size_t>(pl.TT) * IC * OC;
            float* V = scratch;  // plain fp32; the TensorGEMM makes the TF32 hi/lo split on chip
            float* Mbuf = scratch + v_plane;
            for (int R0 = 0; R0 < pl.total_tile_rows; R0 += pl.rows_per_chunk) {
                const int R1 = R0 + pl.rows_per_chunk < pl.total_tile_rows ? R0 + pl.rows_per_chunk : pl.total_tile_rows;
                const int Tc = (R1 - R0) * pl.wg.tilesX;
                if ((rc = wino_input_transform(pl.tile, input, V, pl.wg, R0, R1, s))) return rc;
                GemmProblem g{};
                g.A = V;
                g.B_hi = packed; g.B_lo = pl.np == 2 ? packed + u_plane : nullptr;
                g.D = Mbuf;
                g.M = Tc; g.N = OC; g.K = IC; g.G = pl.TT;
                g.planes = pl.np; g.epilogue = EPI_ROWMAJOR; g.ldd = OC; g.split_k = 1;
                // algorithmic (direct-conv, booster.h:145-148) FLOPs of the output rows this chunk covers
                g.algo_flops = 2.0 * OC * IC * 9.0 * p->output_h * p->output_w * batch *
                               (static_cast<double>(R1 - R0) / pl.total_tile_rows);
                if ((rc = tensor_gemm(g, s))) return rc;
                if ((rc = wino_output_transform(pl.tile, Mbuf, output, b, pl.wg, R0, R1, relu, pool, s))) return rc;
            }
            return 0;
        }
        case FCUDA_IM2COL: {
            if (pool) return -200;
            const size_t w_plane = static_cast<size_t>(OC) * pl.pg.Kp;
            float* P = scratch;
            for (long long m0 = 0; m0 < pl.total_pixels; m0 += pl.pixels_per_chunk) {
                const int rows = static_cast<int>(m0 + pl.pixels_per_chunk < pl.total_pixels ? pl.pixels_per_chunk
                                                                                               : pl.total_pixels - m0);
                if ((rc = im2col_pack(input, P, nullptr, pl.pg, m0, rows, s))) return rc;
                GemmProblem g{};
                g.A = P;
                g.B_hi = packed; g.B_lo = pl.np == 2 ? packed + w_plane : nullptr;
                g.D = output;
                g.M = rows; g.N = OC; g.K = pl.pg.Kp; g.G = 1;
                g.planes = pl.np; g.epilogue = EPI_NCHW; g.P = p->output_h * p->output_w; g.m_offset = m0;
                g.bias = b; g.relu = relu; g.split_k = 1;
                g.algo_flops = 2.0 * OC * pl.pg.K * static_cast<double>(rows);
                if ((rc = tensor_gemm(g, s))) return rc;
            }
            return 0;
        }
        case FCUDA_SGECONV: {
            const int taps = p->kernel_h * p->kernel_w;
            const int G = p->group > 0 ? p->group : 1;
            const int ICg = IC / G, OCg = OC / G;
            const size_t wplane = conv_igemm_packed_floats(OCg, ICg, taps, 1);
            const size_t wgroup = conv_igemm_packed_floats(OCg, ICg, taps, pl.np);
            const size_t in_plane = static_cast<size_t>(p->input_h) * p->input_w;
            const size_t out_plane = static_cast<size_t>(p->output_h) * p->output_w;
            for (int gi = 0; gi < G; ++gi) {  // one launch per group on channel slices (G == 1: the whole tensor)
                IgemmProblem g{};
                const float* wg = packed + static_cast<size_t>(gi) * wgroup;
                g.input = input + static_cast<size_t>(gi) * ICg * in_plane;
                g.w_hi = wg;
                g.w_lo = pl.np == 2 ? wg + wplane : nullptr;
                g.bias = b ? b + static_cast<size_t>(gi) * OCg : nullptr;
                g.output = output + static_cast<size_t>(gi) * OCg * out_plane;
                g.residual = residual ? residual + static_cast<size_t>(gi) * OCg * out_plane : nullptr;
                g.N = batch; g.IC = ICg; g.OC = OCg;
                g.in_c_total = IC; g.out_c_total = OC;
                g.KH = p->kernel_h; g.KW = p->kernel_w; g.pad_top = p->pad_top; g.pad_left = p->pad_left;
                g.stride_h = p->stride_h; g.stride_w = p->stride_w;
                g.dil_h = dil_h; g.dil_w = dil_w;
                if (taps == 1 && p->pad_top == 0 && p->pad_left == 0 && p->stride_h == 1 && p->stride_w == 1) {
                    // pointwise stride 1: address each image as one H*W-long row (fuller 32-pixel boxes)
                    g.H = 1; g.W = p->input_h * p->input_w; g.OH = 1; g.OW = p->output_h * p->output_w;
                } else {
                    g.H = p->input_h; g.W = p->input_w; g.OH = p->output_h; g.OW = p->output_w;
                }
                g.planes = igemm_planes(); g.relu = residual ? relu_after_add : relu;
                g.pool = pool;
                if (pool) {  // pooled output planes
                    g.output = output + static_cast<size_t>(gi) * OCg * (static_cast<size_t>((p->output_h + 1) / 2) * ((p->output_w + 1) / 2));
                    g.out_c_total = OC;
                }
                if ((rc = conv_igemm_forward(g, s))) return rc;
            }
            return 0;
        }
        case FCUDA_NAIVE:
            if (pool) return -200;
            return conv_direct(input, packed, b, output, pl.pg, OC, relu, batch, s);
        case FCUDA_DEPTHWISE:
            if (pool) return -200;
            return depthwise_forward(input, packed, b, output, pl.dg, relu, batch, s);
        default:
            return -1;
    }
}

// Can fcuda_conv_forward_pool fuse the pooling for this layer?  Winograd: always (the output tile starts at an even
// coordinate); implicit GEMM: the 3x3 / stride-1 slab kernel (group 1).
int fcuda_conv_can_pool(const FcudaConvParam* p, int algo) {
    if (!p) return 0;
    if (algo == FCUDA_WINOGRADF63 || algo == FCUDA_WINOGRADF23) return 1;
    if (algo == FCUDA_SGECONV) {
        IgemmProblem g{};
        g.IC = p->input_channels / (p->group > 0 ? p->group : 1);
        g.KH = p->kernel_h; g.KW = p->kernel_w; g.stride_h = p->stride_h; g.stride_w = p->stride_w;
        g.pad_top = p->pad_top; g.pad_left = p->pad_left;
        g.H = p->input_h; g.W = p->input_w;
        return conv_igemm_can_pool(g) ? 1 : 0;
    }
    return 0;
}

int fcuda_igemm_halo_tile(const FcudaConvParam* p, int* geom) {
    if (!p) return 0;
    IgemmProblem g{};
    const int G = p->group > 0 ? p->group : 1;
    g.N = 1; g.IC = p->input_channels / G; g.OC = p->output_channels / G;
    g.H = p->input_h; g.W = p->input_w; g.OH = p->output_h; g.OW = p->output_w;
    g.KH = p->kernel_h; g.KW = p->kernel_w; g.stride_h = p->stride_h; g.stride_w = p->stride_w;
    g.pad_top = p->pad_top; g.pad_left = p->pad_left;
    g.planes = igemm_planes();
    HaloGeom hg;
    if (!conv_igemm_halo_geometry(g, &hg)) return 0;
    if (geom) { geom[0] = hg.R; geom[1] = hg.C; geom[2] = hg.Rb; geom[3] = hg.Cb; }
    return 1;
}

int fcuda_igemm_presplit_tile(const FcudaConvParam* p, int* geom) {
    if (!p) return 0;
    IgemmProblem g{};
    const int G = p->group > 0 ? p->group : 1;
    g.N = 1; g.IC = p->input_channels / G; g.OC = p->output_channels / G;
    g.H = p->input_h; g.W = p->input_w; g.OH = p->output_h; g.OW = p->output_w;
    g.KH = p->kernel_h; g.KW = p->kernel_w; g.stride_h = p->stride_h; g.stride_w = p->stride_w;
    g.pad_top = p->pad_top; g.pad_left = p->pad_left;
    g.planes = igemm_planes();
    HaloGeom hg;
    if (!conv_igemm_presplit_geometry(g, &hg)) return 0;
    if (geom) { geom[0] = hg.R; geom[1] = hg.C; geom[2] = hg.Rb; geom[3] = hg.Cb; }
    return 1;
}

int fcuda_conv_forward_pool(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                            float* scratch, const float* bias, int batch, void* stream) {
    if (!p) return -100;
    if (!fcuda_conv_can_pool(p, algo)) return -200;
    return conv_forward_impl(p, algo, output, input, packed, scratch, bias, nullptr, 0, batch, stream, 1, 1, 1);
}

int fcuda_tensor_gemm(float* d, const float* a, const float* b_hi, const float* b_lo, int m, int n, int k, int g,
                      void* stream) {
    GemmProblem p{};
    p.A = a; p.B_hi = b_hi; p.B_lo = b_lo; p.D = d;
    p.M = m; p.N = n; p.K = k; p.G = g;
    p.planes = b_lo ? 2 : 1;
    p.epilogue = EPI_ROWMAJOR; p.ldd = n; p.split_k = 1;
    return tensor_gemm(p, as_stream(stream));
}

int fcuda_split_tf32(float* hi, float* lo, const float* x, size_t n, void* stream) {
    return split_tf32_planes(x, hi, lo, n, as_stream(stream));
}

// ---------------------------------------------------------------------------------------------
// InnerProduct
// ---------------------------------------------------------------------------------------------
static bool fc_tensor_path(int input_size) { return input_size % 4 == 0; }

// weight streaming is HBM-bound: split K until there are ~2 CTAs per SM; every split owns >= 8 k-blocks
static int fc_split(int input_size, int output_size, int batch) {
    if (!fc_tensor_path(input_size)) return 1;
    const int num_m = ceil_div(output_size, 128) * ceil_div(batch, 128);
    int split = ceil_div(2 * sm_count(), num_m);
    const int kb = ceil_div(input_size, 32);
    if (split > kb / 8) split = kb / 8;
    if (split > 64) split = 64;
    if (split < 1) split = 1;
    return tensor_gemm_effective_split(input_size, split);
}

int fcuda_inner_product_get_buffer_size(int input_size, int output_size, int batch, size_t* scratch_floats,
                                        size_t* packed_kernel_floats) {
    if (input_size <= 0 || output_size <= 0 || batch < 1) return -100;
    const int np = fc_tensor_path(input_size) ? planes() : 1;
    // W (the streamed operand) is kept once as plain fp32; only the small activation matrix gets hi/lo planes.
    // scratch = [X_hi | X_lo] (3xTF32 mode) + one partial-sum plane (batch x out) per k-split
    if (packed_kernel_floats) *packed_kernel_floats = static_cast<size_t>(output_size) * input_size;
    if (scratch_floats)
        *scratch_floats = (np == 2 ? 2 * static_cast<size_t>(batch) * input_size : 0) +
                          static_cast<size_t>(fc_split(input_size, output_size, batch)) * batch * output_size;
    return 0;
}

int fcuda_inner_product_init(int input_size, int output_size, float* packed, const float* raw, void* stream) {
    if (input_size <= 0 || output_size <= 0 || !packed || !raw) return -100;
    cudaStream_t s = as_stream(stream);
    const size_t n = static_cast<size_t>(output_size) * input_size;
    const float* d_raw;
    float* tmp;
    int rc = stage_to_device(raw, n, &d_raw, &tmp, s);
    if (rc) return rc;
    if (cudaMemcpyAsync(packed, d_raw, n * sizeof(float), cudaMemcpyDeviceToDevice, s) != cudaSuccess) rc = FCUDA_ERR_CUDA;
    if (tmp) {
        cudaStreamSynchronize(s);
        cudaFree(tmp);
    }
    return rc;
}

int fcuda_inner_product_forward(int input_size, int output_size, float* output, const float* input,
                                const float* packed, const float* bias, float* scratch, int relu, int batch,
                                void* stream) {
    if (input_size <= 0 || output_size <= 0 || batch < 1 || !output || !input || !packed || !scratch) return -100;
    cudaStream_t s = as_stream(stream);
    const bool tc = fc_tensor_path(input_size);
    const int np = tc ? planes() : 1;
    const size_t xn = static_cast<size_t>(batch) * input_size;
    float* part = scratch + (np == 2 ? 2 * xn : 0);  // [split][batch][out]
    int rc;
    GemmProblem g{};
    g.A = packed;  // A = W (out x in), plain fp32: output features on the 128-row M side
    g.B_hi = input; g.B_lo = nullptr;                           // B = X (batch x in)
    if (np == 2) {
        if ((rc = split_tf32_planes(input, scratch, scratch + xn, xn, s))) return rc;
        g.B_hi = scratch; g.B_lo = scratch + xn;
    }
    g.D = part;
    g.M = output_size; g.N = batch; g.K = input_size; g.G = 1;
    g.planes = np; g.epilogue = EPI_COLMAJOR_PARTIAL; g.ldd = output_size;
    g.split_stride = static_cast<long long>(batch) * output_size;
    g.split_k = fc_split(input_size, output_size, batch);
    g.algo_flops = 2.0 * output_size * static_cast<double>(input_size) * batch;
    if (tc && tensor_gemm_supported(g)) rc = tensor_gemm(g, s);
    else { g.split_k = 1; rc = simt_gemm(g, s); count_launch(); }
    if (rc) return rc;
    // fixed-order sum of the k-split planes + bias + ReLU: deterministic (sgemv.cpp:334-395 is a plain ordered dot product)
    return fc_reduce(output, part, bias, g.split_k, output_size, batch, relu, s);
}

// ---------------------------------------------------------------------------------------------
// Remaining layers
// ---------------------------------------------------------------------------------------------
int fcuda_pooling_out_dim(int in, int pad_a, int pad_b, int kernel, int stride) {
    // pooling_layer.h:129-130
    return static_cast<int>(ceilf(static_cast<float>(in + pad_a + pad_b - kernel) / static_cast<float>(stride))) + 1;
}

int fcuda_pooling_forward(float* output, const float* input, int channels, int in_h, int in_w, int type, int kernel_h,
                          int kernel_w, int stride_h, int stride_w, int pad_left, int pad_right, int pad_top,
                          int pad_bottom, int global_pooling, int batch, void* stream) {
    if (!output || !input || channels <= 0 || in_h <= 0 || in_w <= 0 || batch < 1) return -100;
    PoolGeom g;
    g.H = in_h; g.W = in_w; g.type = type;
    g.stride_h = stride_h > 0 ? stride_h : 1; g.stride_w = stride_w > 0 ? stride_w : 1;
    g.pad_left = pad_left; g.pad_right = pad_right; g.pad_top = pad_top; g.pad_bottom = pad_bottom;
    if (global_pooling) {  // pooling_layer.h:114-121
        g.KH = in_h; g.KW = in_w; g.OH = 1; g.OW = 1;
    } else {
        if (kernel_h <= 0 || kernel_w <= 0) return -100;
        g.KH = kernel_h; g.KW = kernel_w;
        g.OH = fcuda_pooling_out_dim(in_h, pad_top, pad_bottom, kernel_h, g.stride_h);
        g.OW = fcuda_pooling_out_dim(in_w, pad_left, pad_right, kernel_w, g.stride_w);
    }
    return pooling_forward(input, output, g, channels, batch, as_stream(stream));
}

int fcuda_batchnorm_forward(float* output, const float* input, int channels, size_t stride, const float* alpha,
                            const float* beta, const float* scale, const float* scale_bias, int relu, int batch,
                            void* stream) {
    if (!output || !input || !alpha || !beta || channels <= 0) return -100;
    return channel_affine(input, output, channels, stride, beta, alpha, scale, scale_bias, relu, batch, as_stream(stream));
}

int fcuda_scale_forward(float* output, const float* input, int channels, size_t stride, const float* scale,
                        const float* bias, int batch, void* stream) {
    if (!output || !input || !scale || channels <= 0) return -100;
    return channel_affine(input, output, channels, stride, scale, bias, nullptr, nullptr, 0, batch, as_stream(stream));
}

int fcuda_eltwise_add_forward(float* output, const float* a, const float* b, size_t n, int relu, void* stream) {
    if (!output || !a || !b) return -100;
    return add_relu(a, b, output, n, relu, as_stream(stream));
}

int fcuda_eltwise_forward(float* output, const float* a, const float* b, size_t n, int op, float coeff_a, float coeff_b,
                          int relu, void* stream) {
    if (!output || !a || !b) return -100;
    if (op < 0 || op > 2) return -200;
    if (op == 1 && coeff_a == 1.f && coeff_b == 1.f) return add_relu(a, b, output, n, relu, as_stream(stream));
    return eltwise(a, b, output, n, op, coeff_a, coeff_b, relu, as_stream(stream));
}

int fcuda_relu_forward(float* output, const float* input, size_t n, void* stream) {
    if (!output || !input) return -100;
    return scale_relu(input, output, n, 1.f, 1, as_stream(stream));
}

int fcuda_softmax_forward(float* output, const float* input, size_t n_per_image, int batch, void* stream) {
    if (!output || !input || batch < 1) return -100;
    return softmax_forward(input, output, n_per_image, batch, as_stream(stream));
}

int fcuda_dropout_forward(float* output, const float* input, size_t n, float scale, void* stream) {
    if (!output || !input) return -100;
    return scale_relu(input, output, n, scale, 0, as_stream(stream));
}

int fcuda_copy_channels(float* dst, int dst_channels, int dst_channel_offset, const float* src, int channels,
                        size_t stride, int batch, void* stream) {
    if (!dst || !src || channels <= 0 || dst_channel_offset < 0 || dst_channel_offset + channels > dst_channels)
        return -100;
    return copy_channels(src, dst, static_cast<size_t>(channels) * stride, static_cast<size_t>(dst_channels) * stride,
                         static_cast<size_t>(dst_channel_offset) * stride, batch, as_stream(stream));
}

int fcuda_pixel_channels(int type, int* src_channels, int* out_channels) { return pixel_channels(type, src_channels, out_channels); }

int fcuda_from_pixels(float* output, const unsigned char* pixels, int type, int w, int h, int target_w, int target_h,
                      const float* mean_vals, const float* norm_vals, int batch, void* stream) {
    if (!output || !pixels) return -100;
    return from_pixels(output, pixels, type, w, h, target_w, target_h, mean_vals, norm_vals, batch, as_stream(stream));
}

int fcuda_set_tuning(const char* name, int value) { return tune_set(name, value); }
int fcuda_get_tuning(const char* name) {
    for (int k = 0; k < TUNE_COUNT; ++k)
        if (name && !strcmp(name, tune_name(k))) return tune_get(k);
    return -200;
}

void fcuda_profile_tensor_gemm(int enable) { gemm_profile_enable(enable != 0); }
int fcuda_profile_collect_kind(int kind, double* total_ms, double* algo_flops, double* mma_flops, double* algo_bytes,
                               long long* launches) {
    profile_collect_kind(kind, total_ms, algo_flops, mma_flops, algo_bytes, launches);
    return 0;
}
int fcuda_profile_collect(double* total_ms, double* algo_flops, double* mma_flops, long long* launches) {
    gemm_profile_collect(total_ms, algo_flops, mma_flops, launches);
    return 0;
}

unsigned long long fcuda_launch_count(void) { return launch_count(); }
void fcuda_reset_launch_count(void) { reset_launch_count(); }

}  // extern "C"
