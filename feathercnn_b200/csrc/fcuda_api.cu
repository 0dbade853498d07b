// extern "C" surface of libfcuda.so (include/fcuda.h): algorithm selection, workspace planning and the
// per-layer dispatch that stands where booster::ConvBooster's function table stood
// (/root/reference/src/booster/avx/booster.cpp:283-355).
#include "fcuda.h"

#include "activation.cuh"
#include "attention.cuh"
#include "binary_op.cuh"
#include "common.cuh"
#include "conv_direct.cuh"
#include "conv_igemm.cuh"
#include "deconv.cuh"
#include "depthwise.cuh"
#include "detection.cuh"
#include "instance_norm.cuh"
#include "layer_norm.cuh"
#include "layers.cuh"
#include "lrn.cuh"
#include "normalize.cuh"
#include "pack.cuh"
#include "preprocess.cuh"
#include "resize.cuh"
#include "route.cuh"
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

int interp_check_and_size(FcudaInterpParam* p) {
    if (!p) return -100;
    if (p->resize_type != 1 && p->resize_type != 2) return -200;
    if (p->input_h <= 0 || p->input_w <= 0 || p->output_height < 0 || p->output_width < 0) return -100;
    const bool sized = p->output_height > 0 && p->output_width > 0;
    // the scales are read where they size the output, and by nearest where its explicit size is absent
    const bool scale_h_used = !sized || (p->resize_type == 1 && !p->output_height);
    const bool scale_w_used = !sized || (p->resize_type == 1 && !p->output_width);
    if ((scale_h_used && !(p->height_scale > 0.f)) || (scale_w_used && !(p->width_scale > 0.f))) return -100;
    long long oh = p->output_height, ow = p->output_width;
    if (!sized) {  // ncnn: static_cast<int>(h * height_scale), an fp32 product
        const float fh = static_cast<float>(p->input_h) * p->height_scale;
        const float fw = static_cast<float>(p->input_w) * p->width_scale;
        if (!(fh < 2147483648.f) || !(fw < 2147483648.f)) return -100;
        oh = static_cast<long long>(fh);
        ow = static_cast<long long>(fw);
    }
    if (oh <= 0 || ow <= 0 || oh * ow > 0x7fffffffLL || static_cast<long long>(p->input_h) * p->input_w > 0x7fffffffLL)
        return -100;
    p->output_h = static_cast<int>(oh);
    p->output_w = static_cast<int>(ow);
    return 0;
}

// The fp32 source-coordinate scale of one axis (include/fcuda.h, fcuda_interp_forward)
float interp_scale(const FcudaInterpParam& p, int in, int out, int explicit_out, float scale) {
    if (p.resize_type == 1) return explicit_out ? static_cast<float>(in) / static_cast<float>(out) : 1.f / scale;
    if (p.align_corner) return out > 1 ? static_cast<float>(in - 1) / static_cast<float>(out - 1) : 0.f;
    return static_cast<float>(in) / static_cast<float>(out);
}

// Prior count of one feature-map location (include/fcuda.h, fcuda_priorbox_forward); -200 outside the limits.
int priorbox_count(const FcudaPriorBoxParam* p, int* per_loc) {
    if (!p) return -100;
    if (p->num_min_sizes < 1 || p->num_min_sizes > FCUDA_PRIORBOX_MAX || p->num_aspect_ratios < 0 ||
        p->num_aspect_ratios > FCUDA_PRIORBOX_MAX || (p->num_max_sizes != 0 && p->num_max_sizes != p->num_min_sizes))
        return -200;
    int ars = 0;
    for (int a = 0; a < p->num_aspect_ratios; ++a) {
        if (!(p->aspect_ratios[a] > 0.f) || !isfinite(p->aspect_ratios[a])) return -200;
        ars += fabsf(p->aspect_ratios[a] - 1.f) < 1e-6f ? 0 : (p->flip ? 2 : 1);
    }
    for (int k = 0; k < p->num_min_sizes; ++k) {
        if (!(p->min_sizes[k] > 0.f) || !isfinite(p->min_sizes[k])) return -200;
        if (p->num_max_sizes && !(p->max_sizes[k] > p->min_sizes[k] && isfinite(p->max_sizes[k]))) return -200;
    }
    if (!isfinite(p->offset) || !isfinite(p->step_w) || !isfinite(p->step_h)) return -200;
    *per_loc = p->num_min_sizes * (1 + (p->num_max_sizes ? 1 : 0) + ars);
    return 0;
}

constexpr long long kMaxPriors = 1LL << 24;

int detection_limits(int P, int C, int nms_top_k, int batch) {
    if (P < 1 || C < 1 || batch < 1) return -100;
    if (P >= kMaxPriors || C > 1024 || nms_top_k < 1 || nms_top_k > 1024 || batch > 65535) return -200;
    return 0;
}

// Limits of the YOLO head (include/fcuda.h, FcudaYoloParam): -100 / -200, and the slot count when both pass.
int yolo_limits(const FcudaYoloParam* p, int batch, int* slots) {
    if (!p) return -100;
    const bool v3 = p->version == 3;
    if ((p->version != 2 && !v3) || p->num_class < 1 || p->num_class > 1024 || p->num_box < 1 ||
        p->num_box > FCUDA_YOLO_MAX_BOXES || p->num_scales < 1 || p->num_scales > (v3 ? FCUDA_YOLO_MAX_SCALES : 1) ||
        p->num_biases < 0 || p->num_biases > FCUDA_YOLO_MAX_BIASES || (!v3 && p->num_biases < 2 * p->num_box) ||
        p->nms_top_k < 1 || p->nms_top_k > 1024 || p->keep_top_k < 1 || p->keep_top_k > 1024 || isnan(p->nms_threshold))
        return -200;
    if (v3) {
        for (int k = 0; k < p->num_scales * p->num_box; ++k)
            if (p->mask[k] < 0 || p->mask[k] >= p->num_biases / 2) return -200;
        for (int b = 0; b < p->num_scales; ++b)
            if (!(p->anchors_scale[b] > 0.f)) return -200;
    }
    if (batch < 1) return -100;
    if (batch > 65535) return -200;
    long long total = 0;
    for (int b = 0; b < p->num_scales; ++b) {
        if (p->grid_h[b] < 1 || p->grid_w[b] < 1) return -100;
        // the fp32 products anchors_scale * side must truncate to an int (NaN and inf fail too)
        const int side = p->grid_h[b] > p->grid_w[b] ? p->grid_h[b] : p->grid_w[b];
        if (v3 && !(p->anchors_scale[b] * static_cast<float>(side) < 2147483520.f)) return -200;
        total += static_cast<long long>(p->num_box) * p->grid_h[b] * p->grid_w[b];
        if (total >= kMaxPriors) return -200;
    }
    *slots = static_cast<int>(total);
    return 0;
}

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
            g.dil_h = 1; g.dil_w = 1;  // conv_launch sets the layer's
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

// The launches of one planned convolution; `epi` is what every kernel applies after its contraction (epi.pool only on
// the algorithms of fcuda_conv_can_pool).
static int conv_launch(const FcudaConvParam* p, const ConvPlan& pl, float* output, const float* input, const float* packed,
                       float* scratch, const ConvEpilogue& epi, int dil_h, int dil_w, int batch, cudaStream_t s) {
    int rc;
    const int IC = p->input_channels, OC = p->output_channels;
    switch (pl.algo) {
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
                if ((rc = wino_output_transform(pl.tile, Mbuf, output, pl.wg, R0, R1, epi, s))) return rc;
            }
            return 0;
        }
        case FCUDA_IM2COL: {
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
                g.epi = epi; g.split_k = 1;
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
            const size_t out_plane = epi.pool ? static_cast<size_t>((p->output_h + 1) / 2) * ((p->output_w + 1) / 2)
                                              : static_cast<size_t>(p->output_h) * p->output_w;
            for (int gi = 0; gi < G; ++gi) {  // one launch per group on channel slices (G == 1: the whole tensor)
                IgemmProblem g{};
                const float* wg = packed + static_cast<size_t>(gi) * wgroup;
                g.input = input + static_cast<size_t>(gi) * ICg * in_plane;
                g.w_hi = wg;
                g.w_lo = pl.np == 2 ? wg + wplane : nullptr;
                g.output = output + static_cast<size_t>(gi) * OCg * out_plane;
                g.epi = epi;
                if (epi.bias) g.epi.bias += static_cast<size_t>(gi) * OCg;
                if (epi.residual) g.epi.residual += static_cast<size_t>(gi) * OCg * out_plane;
                g.N = batch; g.IC = ICg; g.OC = OCg;
                g.in_c_total = IC; g.out_c_total = OC;
                g.KH = p->kernel_h; g.KW = p->kernel_w; g.pad_top = p->pad_top; g.pad_left = p->pad_left;
                g.stride_h = p->stride_h; g.stride_w = p->stride_w;
                g.dil_h = dil_h; g.dil_w = dil_w;
                if (taps == 1 && p->pad_top == 0 && p->pad_left == 0 && p->stride_h == 1 && p->stride_w == 1 &&
                    p->output_h == p->input_h && p->output_w == p->input_w) {
                    // pointwise stride 1, no padding: address each image as one H*W-long row (fuller 32-pixel boxes)
                    g.H = 1; g.W = p->input_h * p->input_w; g.OH = 1; g.OW = p->output_h * p->output_w;
                } else {
                    g.H = p->input_h; g.W = p->input_w; g.OH = p->output_h; g.OW = p->output_w;
                }
                g.planes = igemm_planes();
                if ((rc = conv_igemm_forward(g, s))) return rc;
            }
            return 0;
        }
        case FCUDA_NAIVE:
            return conv_direct(input, packed, output, pl.pg, OC, epi, batch, s);
        case FCUDA_DEPTHWISE: {
            DwGeom g = pl.dg;
            g.dil_h = dil_h; g.dil_w = dil_w;
            return depthwise_forward(input, packed, output, g, epi, batch, s);
        }
        default:
            return -1;
    }
}

// The one forward path: fcuda_conv_forward_opts, and the five older entry points with the options their signatures carry
// (include/fcuda.h, FcudaConvOptions).  clip_bounds_given is false from the entry points without clip bounds: for them a
// Clip activation is refused, after the plan's own error and before the tensor checks.
static int conv_forward(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                        float* scratch, const float* bias, const FcudaConvOptions& o, bool clip_bounds_given, int batch,
                        void* stream) {
    if (!p || o.dilation_h < 0 || o.dilation_w < 0) return -100;
    const int dil_h = o.dilation_h ? o.dilation_h : 1, dil_w = o.dilation_w ? o.dilation_w : 1;
    const bool dilated = dil_h > 1 || dil_w > 1;
    const bool clip = clip_bounds_given && p->activation == FCUDA_ACT_CLIP;
    if (clip && !(o.clip_min <= o.clip_max)) return -200;  // (a NaN bound too)
    if (clip_bounds_given && !clip && (o.clip_min != 0.f || o.clip_max != 0.f)) return -200;  // bounds without a Clip
    if (dilated && algo != FCUDA_SGECONV && algo != FCUDA_DEPTHWISE) return -200;  // only these space their taps
    // The implicit GEMM adds the residual in its epilogue when the convolution has no activation of its own; every other
    // case is the convolution, then the reference's add_relu in place.
    const bool fuse_residual = o.residual && algo == FCUDA_SGECONV && p->activation == FCUDA_ACT_NONE;
    if (dilated && o.residual && !fuse_residual) return -200;
    if (o.pool && !fcuda_conv_can_pool(p, algo)) return -200;
    // not built (a dilated depthwise clamps in its epilogue like an undilated one)
    if ((clip && (o.residual || (dilated && algo != FCUDA_DEPTHWISE) || o.pool)) || (o.pool && (o.residual || dilated))) return -200;
    ConvPlan pl;
    int rc = make_plan(p, algo, batch, &pl);
    if (rc) return rc;
    if (p->activation == FCUDA_ACT_CLIP && !clip_bounds_given) return -200;
    if (!output || !input || !packed) return -100;
    if (pl.scratch_floats && !scratch) return -100;
    const ConvEpilogue epi = conv_epilogue(p->activation, p->bias_term, bias, o.clip_min, o.clip_max,
                                           fuse_residual ? o.residual : nullptr, o.relu_after_add, o.pool);
    if ((rc = conv_launch(p, pl, output, input, packed, scratch, epi, dil_h, dil_w, batch, as_stream(stream)))) return rc;
    if (!o.residual || fuse_residual) return 0;
    const size_t n = static_cast<size_t>(batch) * p->output_channels * p->output_h * p->output_w;
    return add_relu(output, o.residual, output, n, o.relu_after_add, as_stream(stream));
}

int fcuda_conv_forward_opts(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                            float* scratch, const float* bias, const FcudaConvOptions* options, int batch, void* stream) {
    return conv_forward(p, algo, output, input, packed, scratch, bias, options ? *options : FcudaConvOptions{}, true, batch,
                        stream);
}

int fcuda_conv_forward(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                       float* scratch, const float* bias, int batch, void* stream) {
    return conv_forward(p, algo, output, input, packed, scratch, bias, FcudaConvOptions{}, false, batch, stream);
}

int fcuda_conv_forward_clip(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                            float* scratch, const float* bias, float clip_min, float clip_max, int batch, void* stream) {
    if (!p) return -100;
    if (p->activation != FCUDA_ACT_CLIP) return -200;
    FcudaConvOptions o{};
    o.clip_min = clip_min; o.clip_max = clip_max;
    return conv_forward(p, algo, output, input, packed, scratch, bias, o, true, batch, stream);
}

int fcuda_conv_forward_residual(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                                float* scratch, const float* bias, const float* residual, int relu_after_add, int batch,
                                void* stream) {
    if (!p || !residual) return -100;
    FcudaConvOptions o{};
    o.residual = residual; o.relu_after_add = relu_after_add;
    return conv_forward(p, algo, output, input, packed, scratch, bias, o, false, batch, stream);
}

int fcuda_conv_forward_pool(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                            float* scratch, const float* bias, int batch, void* stream) {
    FcudaConvOptions o{};
    o.pool = 1;
    return conv_forward(p, algo, output, input, packed, scratch, bias, o, false, batch, stream);
}

int fcuda_conv_forward_ext(const FcudaConvParam* p, int algo, float* output, const float* input, const float* packed,
                           float* scratch, const float* bias, const float* residual, int relu_after_add, int dilation_h,
                           int dilation_w, int batch, void* stream) {
    if (!p || dilation_h < 1 || dilation_w < 1) return -100;
    FcudaConvOptions o{};
    o.residual = residual; o.relu_after_add = relu_after_add;
    o.dilation_h = dilation_h; o.dilation_w = dilation_w;
    return conv_forward(p, algo, output, input, packed, scratch, bias, o, false, batch, stream);
}

// The implicit-GEMM problem of one group of a layer, without tensors (N = 1): what the tile and pooling queries read
static IgemmProblem igemm_problem(const FcudaConvParam* p) {
    IgemmProblem g{};
    const int G = p->group > 0 ? p->group : 1;
    g.N = 1; g.IC = p->input_channels / G; g.OC = p->output_channels / G;
    g.H = p->input_h; g.W = p->input_w; g.OH = p->output_h; g.OW = p->output_w;
    g.KH = p->kernel_h; g.KW = p->kernel_w; g.stride_h = p->stride_h; g.stride_w = p->stride_w;
    g.pad_top = p->pad_top; g.pad_left = p->pad_left;
    g.planes = igemm_planes();
    return g;
}

// Can the epilogue fuse the pooling (FcudaConvOptions::pool) for this layer?  Winograd: always (the output tile starts at an even
// coordinate); implicit GEMM: the 3x3 / stride-1 slab kernel (group 1).
int fcuda_conv_can_pool(const FcudaConvParam* p, int algo) {
    if (!p) return 0;
    if (algo == FCUDA_WINOGRADF63 || algo == FCUDA_WINOGRADF23) return 1;
    if (algo == FCUDA_SGECONV) return conv_igemm_can_pool(igemm_problem(p)) ? 1 : 0;
    return 0;
}

static int igemm_tile(const FcudaConvParam* p, int* geom, bool (*geometry)(const IgemmProblem&, HaloGeom*)) {
    if (!p) return 0;
    HaloGeom hg;
    if (!geometry(igemm_problem(p), &hg)) return 0;
    if (geom) { geom[0] = hg.R; geom[1] = hg.C; geom[2] = hg.Rb; geom[3] = hg.Cb; }
    return 1;
}

int fcuda_igemm_halo_tile(const FcudaConvParam* p, int* geom) { return igemm_tile(p, geom, conv_igemm_halo_geometry); }
int fcuda_igemm_presplit_tile(const FcudaConvParam* p, int* geom) { return igemm_tile(p, geom, conv_igemm_presplit_geometry); }
int fcuda_igemm_wide_tile(const FcudaConvParam* p, int* geom) { return igemm_tile(p, geom, conv_igemm_wide_geometry); }

int fcuda_igemm_stem_supported(const FcudaConvParam* p, const FcudaConvOptions* o) {
    if (!p) return 0;
    IgemmProblem g = igemm_problem(p);
    if (o) {
        g.epi.residual = o->residual;
        g.epi.pool = o->pool ? 1 : 0;
        g.dil_h = o->dilation_h; g.dil_w = o->dilation_w;
    }
    return conv_igemm_stem_supported(g) ? 1 : 0;
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

int fcuda_binary_op_shape(int a_rank, const int* a_shape, int b_rank, const int* b_shape, int* out_rank, int* out_shape,
                          int* a_aligned, int* b_aligned) {
    if (!a_shape || !b_shape || !out_rank || !out_shape || !a_aligned || !b_aligned) return -100;
    int a[3], b[3];
    for (int k = 0; k < 3; ++k) {
        a[k] = a_shape[k];
        b[k] = b_shape[k];
        if (a[k] < 1 || b[k] < 1) return -100;
    }
    if (a_rank < 1 || a_rank > 3 || b_rank < 1 || b_rank > 3) return -100;
    if ((a_rank < 3 && a[0] != 1) || (a_rank < 2 && a[1] != 1) || (b_rank < 3 && b[0] != 1) || (b_rank < 2 && b[1] != 1))
        return -100;
    const bool equal = a[0] == b[0] && a[1] == b[1] && a[2] == b[2];
    const bool a_one = a[0] == 1 && a[1] == 1 && a[2] == 1, b_one = b[0] == 1 && b[1] == 1 && b[2] == 1;
    int rank = a_rank > b_rank ? a_rank : b_rank;
    if (equal) {
    } else if (a_one) {
        rank = b_rank;
    } else if (b_one) {
        rank = a_rank;
    } else if (a_rank == 3 && b_rank == 1 && b[2] == a[0]) {  // ncnn's per-channel operand
        b[0] = b[2];
        b[2] = 1;
    } else if (b_rank == 3 && a_rank == 1 && a[2] == b[0]) {
        a[0] = a[2];
        a[2] = 1;
    }
    int out[3];
    for (int k = 0; k < 3; ++k) {
        if (a[k] != b[k] && a[k] != 1 && b[k] != 1) return -200;
        out[k] = a[k] == 1 ? b[k] : a[k];
    }
    *out_rank = rank;
    for (int k = 0; k < 3; ++k) {
        out_shape[k] = out[k];
        a_aligned[k] = a[k];
        b_aligned[k] = b[k];
    }
    return 0;
}

// Element strides of an NCHW operand of shape s along the output's axes: 0 where it broadcasts (extent 1).
static BinaryOperand binary_operand(const float* p, const int* s) {
    const long long w = s[3], hw = static_cast<long long>(s[2]) * w;
    return BinaryOperand{p, s[1] * hw, s[1] == 1 ? 0 : hw, s[2] == 1 ? 0 : w, s[3] == 1 ? 0 : 1};
}

int fcuda_binary_op_forward(float* output, const float* a, const int* a_shape, const float* b, const int* b_shape,
                            float b_scalar, int op, int relu, void* stream) {
    if (!output || !a || !a_shape || (b && !b_shape)) return -100;
    int as[4], bs[4], os[4];
    for (int k = 0; k < 4; ++k) {
        as[k] = a_shape[k];
        bs[k] = b ? b_shape[k] : (k == 0 ? as[0] : 1);
        if (as[k] < 1 || bs[k] < 1) return -100;
    }
    if (op < FCUDA_BINARY_ADD || op > FCUDA_BINARY_RATAN2 || as[0] != bs[0]) return -200;
    os[0] = as[0];
    bool a_bc = false, b_bc = false;
    for (int k = 1; k < 4; ++k) {
        if (as[k] != bs[k] && as[k] != 1 && bs[k] != 1) return -200;
        os[k] = as[k] == 1 ? bs[k] : as[k];
        a_bc = a_bc || as[k] != os[k];
        b_bc = b_bc || bs[k] != os[k];
    }
    if (static_cast<long long>(os[2]) * os[3] > 0x7fffffffLL) return -200;
    if ((output == a && a_bc) || (b && output == b && b_bc)) return -200;
    relu = relu ? 1 : 0;
    const cudaStream_t s = as_stream(stream);
    if (!a_bc && (!b || !b_bc)) {
        const size_t n = static_cast<size_t>(os[0]) * os[1] * os[2] * os[3];
        if (b && op == FCUDA_BINARY_ADD) return add_relu(a, b, output, n, relu, s);  // Eltwise SUM
        return binary_op_same(output, a, b, b_scalar, n, op, relu, s);
    }
    return binary_op_broadcast(output, binary_operand(a, as), binary_operand(b, bs), os[1], os[2], os[3], op, relu, os[0],
                               s);
}

int fcuda_relu_forward(float* output, const float* input, size_t n, void* stream) {
    if (!output || !input) return -100;
    return scale_relu(input, output, n, 1.f, 1, as_stream(stream));
}

int fcuda_clip_forward(float* output, const float* input, size_t n, float min, float max, void* stream) {
    if (!output || !input) return -100;
    if (!(min <= max)) return -200;
    return clip(input, output, n, min, max, as_stream(stream));
}

int fcuda_activation_forward(float* output, const float* input, size_t n, int type, float alpha, float beta,
                             void* stream) {
    if (!output || !input || n == 0) return -100;
    if ((type < FCUDA_ACTIVATION_SIGMOID || type > FCUDA_ACTIVATION_HARDSWISH) && type != FCUDA_ACTIVATION_GELU &&
        type != FCUDA_ACTIVATION_GELU_TANH)
        return -200;
    const bool hard = type == FCUDA_ACTIVATION_HARDSIGMOID || type == FCUDA_ACTIVATION_HARDSWISH;
    if (hard && (alpha == 0.f || !isfinite(alpha) || !isfinite(beta))) return -200;
    // ncnn's HardSigmoid / HardSwish load_param, in fp32
    const float lower = hard ? -beta / alpha : 0.f;
    const float upper = hard ? 1.f / alpha + lower : 0.f;
    return activation(output, input, n, type, alpha, beta, lower, upper, as_stream(stream));
}

int fcuda_layer_norm_forward(float* output, const float* input, int n, long long rows, const float* gamma,
                             const float* beta, float eps, void* stream) {
    if (!output || !input || n < 1 || rows < 1) return -100;
    if (!gamma != !beta || !(eps >= 0.f) || !isfinite(eps)) return -200;
    return layer_norm(output, input, n, rows, gamma, beta, eps, as_stream(stream));
}

// [lo, hi) byte range of the rows a [batch][l][ld] operand reads (cols floats of each row)
static void attn_range(const float* p, int ld, long long rows, int cols, uintptr_t* lo, uintptr_t* hi) {
    *lo = reinterpret_cast<uintptr_t>(p);
    *hi = *lo + (static_cast<uintptr_t>(rows - 1) * ld + cols) * sizeof(float);
}

int fcuda_attention_forward(float* o, const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                            int batch, int heads, int d, int lq, int lk, float scale, void* stream) {
    if (!o || !q || !k || !v || batch < 1 || heads < 1 || lq < 1 || lk < 1) return -100;
    if (d < 16 || d > 128 || d % 16 != 0) return -200;
    const long long e = static_cast<long long>(heads) * d;
    if (e > INT32_MAX || ldq < e || ldk < e || ldv < e) return -200;
    if (static_cast<long long>(heads) * ((lq + 63) / 64) > 65535) return -200;
    if (scale == 0.f || !isfinite(scale)) return -200;
    uintptr_t olo, ohi, lo, hi;
    attn_range(o, static_cast<int>(e), static_cast<long long>(batch) * lq, static_cast<int>(e), &olo, &ohi);
    const struct { const float* p; int ld; int l; } ops[3] = {{q, ldq, lq}, {k, ldk, lk}, {v, ldv, lk}};
    for (const auto& op : ops) {
        attn_range(op.p, op.ld, static_cast<long long>(batch) * op.l, static_cast<int>(e), &lo, &hi);
        if (lo < ohi && olo < hi) return -200;
    }
    return attention(o, q, ldq, k, ldk, v, ldv, batch, heads, d, lq, lk, scale, as_stream(stream));
}

int fcuda_prelu_forward(float* output, const float* input, int channels, size_t plane, const float* slope, int num_slope,
                        int batch, void* stream) {
    if (!output || !input || !slope || channels <= 0 || plane == 0 || batch < 1) return -100;
    if (num_slope != 1 && num_slope != channels) return -200;
    return prelu(input, output, slope, channels, plane, num_slope == 1, batch, as_stream(stream));
}

static int normalize_params_ok(int across_spatial, int across_channel, float eps, int eps_mode) {
    return (across_spatial || across_channel) && eps_mode >= 0 && eps_mode <= 2 && eps >= 0.f;  // NaN eps fails >=
}

int fcuda_normalize_workspace_size(int across_spatial, int across_channel, int channels, size_t plane, int batch,
                                   size_t* floats) {
    if (!floats || channels < 1 || plane == 0 || batch < 1) return -100;
    if (!across_spatial && !across_channel) return -200;
    *floats = normalize_workspace_floats(across_spatial != 0, across_channel != 0, channels, plane, batch);
    return 0;
}

int fcuda_normalize_forward(float* output, const float* input, int channels, size_t plane, const float* scale,
                            int num_scale, int across_spatial, int across_channel, float eps, int eps_mode,
                            float* workspace, int batch, void* stream) {
    if (!output || !input || !scale || channels < 1 || plane == 0 || batch < 1) return -100;
    if ((num_scale != 1 && num_scale != channels) || !normalize_params_ok(across_spatial, across_channel, eps, eps_mode))
        return -200;
    if (across_spatial && !workspace) return -100;
    NormalizeGeom g;
    g.channels = channels;
    g.plane = plane;
    g.batch = batch;
    g.across_spatial = across_spatial != 0;
    g.across_channel = across_channel != 0;
    g.shared = num_scale == 1;
    g.eps = eps;
    g.eps_mode = eps_mode;
    return normalize_forward(input, output, scale, g, workspace, as_stream(stream));
}

// -200 for a pad fcuda.h rejects; *padded tells whether any side is non-zero.
static int plane_pad_check(const FcudaPad* pad, int h, int w, PlanePad* out, int* padded) {
    *out = PlanePad{0, 0, 0, 0, 0, 0.f};
    *padded = 0;
    if (!pad) return 0;
    if (pad->top < 0 || pad->bottom < 0 || pad->left < 0 || pad->right < 0 || pad->type < 0 || pad->type > 2) return -200;
    if (pad->type == 2 && (pad->top >= h || pad->bottom >= h || pad->left >= w || pad->right >= w)) return -200;
    const long long ho = static_cast<long long>(h) + pad->top + pad->bottom;
    const long long wo = static_cast<long long>(w) + pad->left + pad->right;
    if (ho * wo > 0x7fffffffll) return -200;
    *out = PlanePad{pad->top, pad->bottom, pad->left, pad->right, pad->type, pad->value};
    *padded = (pad->top | pad->bottom | pad->left | pad->right) != 0;
    return 0;
}

// InstanceNorm's input and padded output planes: float(S) is exact, and the per-CTA re-combination of a plane's partials
// stays bounded (instance_norm.cu).
static const long long kMaxNormPlane = 1ll << 24;

int fcuda_instance_norm_workspace_size(int channels, size_t plane, int batch, size_t* floats) {
    if (!floats || channels < 1 || plane == 0 || batch < 1) return -100;
    *floats = instance_norm_workspace_floats(channels, plane, batch);
    return 0;
}

int fcuda_instance_norm_forward(float* output, const float* input, int channels, int h, int w, const float* gamma,
                                const float* beta, float eps, int relu, const FcudaPad* pad, float* workspace,
                                int batch, void* stream) {
    if (!output || !input || !workspace || !gamma != !beta || channels < 1 || h < 1 || w < 1 || batch < 1) return -100;
    if (!(eps >= 0.f) || static_cast<long long>(h) * w > kMaxNormPlane) return -200;  // NaN eps fails >=
    PlanePad pd;
    int padded = 0;
    if (plane_pad_check(pad, h, w, &pd, &padded)) return -200;
    if (static_cast<long long>(h + pd.top + pd.bottom) * (w + pd.left + pd.right) > kMaxNormPlane) return -200;
    if (padded && output == input) return -200;
    return instance_norm_forward(input, output, channels, h, w, gamma, beta, eps, relu != 0, padded ? &pd : NULL,
                                 workspace, batch, as_stream(stream));
}

int fcuda_padding_forward(float* output, const float* input, int channels, int h, int w, const FcudaPad* pad, int batch,
                          void* stream) {
    if (!output || !input || !pad || channels < 1 || h < 1 || w < 1 || batch < 1) return -100;
    PlanePad pd;
    int padded = 0;
    if (static_cast<long long>(h) * w > 0x7fffffffll || plane_pad_check(pad, h, w, &pd, &padded)) return -200;
    if (padded && output == input) return -200;
    return padding_forward(input, output, channels, h, w, pd, batch, as_stream(stream));
}

int fcuda_lrn_forward(float* output, const float* input, int channels, int h, int w, int region_type, int local_size,
                      float alpha, float beta, float bias, int batch, void* stream) {
    if (!output || !input || channels < 1 || h < 1 || w < 1 || batch < 1) return -100;
    if (region_type < 0 || region_type > 1 || local_size < 1 || local_size % 2 == 0 || output == input) return -200;
    LrnGeom g;
    g.channels = channels;
    g.h = h;
    g.w = w;
    g.batch = batch;
    g.region = region_type;
    g.local_size = local_size;
    g.alpha = alpha;
    g.beta = beta;
    g.bias = bias;
    return lrn_forward(input, output, g, as_stream(stream));
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

int fcuda_interp_output_dim(FcudaInterpParam* param) { return interp_check_and_size(param); }

int fcuda_interp_forward(const FcudaInterpParam* param, float* output, const float* input, int channels, int batch,
                         void* stream) {
    if (!param) return -100;
    FcudaInterpParam p = *param;
    const int rc = interp_check_and_size(&p);
    if (rc) return rc;
    if (!output || !input || channels <= 0 || batch < 1) return -100;
    InterpGeom g;
    g.H = p.input_h; g.W = p.input_w; g.OH = p.output_h; g.OW = p.output_w;
    g.mode = p.resize_type;
    g.align_corner = p.align_corner != 0;
    g.scale_h = interp_scale(p, p.input_h, p.output_h, p.output_height, p.height_scale);
    g.scale_w = interp_scale(p, p.input_w, p.output_w, p.output_width, p.width_scale);
    return interp_forward(input, output, g, static_cast<long long>(batch) * channels, as_stream(stream));
}

int fcuda_pixel_shuffle_forward(float* output, const float* input, int channels, int h, int w, int r, int mode,
                                const float* addend, const FcudaInterpParam* addend_map, int batch, void* stream) {
    if (!output || !input || (addend && !addend_map) || channels < 1 || h < 1 || w < 1 || batch < 1) return -100;
    if (r < 1 || (mode != 0 && mode != 1) || static_cast<long long>(r) * r > channels || channels % (r * r)) return -200;
    const long long oh = static_cast<long long>(h) * r, ow = static_cast<long long>(w) * r;
    if (oh * ow > 0x7fffffffLL || output == input || (addend && output == addend)) return -200;
    const int oc = channels / (r * r);
    ScatterAddend add{};
    if (addend) {
        FcudaInterpParam p = *addend_map;
        if (p.resize_type != 1) return -200;
        const int rc = interp_check_and_size(&p);
        if (rc) return rc;
        if (p.output_h != oh || p.output_w != ow) return -200;
        add = ScatterAddend{addend, p.input_h, p.input_w, interp_scale(p, p.input_h, p.output_h, p.output_height,
                                                                      p.height_scale),
                            interp_scale(p, p.input_w, p.output_w, p.output_width, p.width_scale)};
    }
    // the sub-pixel scatter of a deconvolution with stride r and no pads, bias or ReLU; mode 0 is group = OC (channel
    // p * r^2 + i * r + j), mode 1 group = 1 (channel (i * r + j) * OC + p)
    DeconvScatterGeom g;
    g.OC = oc; g.group = mode == 0 ? oc : 1; g.stride_h = g.stride_w = r;
    g.Hc = h; g.Wc = w; g.OH = static_cast<int>(oh); g.OW = static_cast<int>(ow); g.pad_top = g.pad_left = 0;
    return deconv_scatter(input, nullptr, output, g, 0, addend ? &add : nullptr, PROF_PIXEL_SHUFFLE, batch,
                          as_stream(stream));
}

int fcuda_crop_forward(float* output, const float* input, int channels, int in_h, int in_w, int coff, int hoff, int woff,
                       int out_c, int out_h, int out_w, int batch, void* stream) {
    if (channels <= 0 || in_h <= 0 || in_w <= 0 || out_c <= 0 || out_h <= 0 || out_w <= 0 || batch < 1 || coff < 0 ||
        hoff < 0 || woff < 0)
        return -100;
    if (static_cast<long long>(coff) + out_c > channels || static_cast<long long>(hoff) + out_h > in_h ||
        static_cast<long long>(woff) + out_w > in_w)
        return -100;
    if (!output || !input) return -100;
    CropGeom g;
    g.C = channels; g.H = in_h; g.W = in_w; g.coff = coff; g.hoff = hoff; g.woff = woff;
    g.OC = out_c; g.OH = out_h; g.OW = out_w;
    return crop_forward(input, output, g, batch, as_stream(stream));
}

int fcuda_permute_forward(float* output, const float* input, int c, int h, int w, int order_type, int batch, void* stream) {
    if (!output || !input || c < 1 || h < 1 || w < 1 || batch < 1) return -100;
    if (order_type < 0 || order_type > 5) return -200;
    return permute_forward(input, output, c, h, w, order_type, batch, as_stream(stream));
}

int fcuda_softmax_axis_forward(float* output, const float* input, int outer, int len, int inner, int batch, void* stream) {
    if (!output || !input || outer < 1 || len < 1 || inner < 1 || batch < 1) return -100;
    return softmax_axis_forward(input, output, outer, len, inner, batch, as_stream(stream));
}

int fcuda_priorbox_per_location(const FcudaPriorBoxParam* param, int* per_location) {
    if (!per_location) return -100;
    return priorbox_count(param, per_location);
}

int fcuda_priorbox_forward(float* output, const FcudaPriorBoxParam* param, int feat_w, int feat_h, int img_w, int img_h,
                           void* stream) {
    int per_loc = 0;
    const int rc = priorbox_count(param, &per_loc);
    if (rc) return rc;
    if (!output || feat_w < 1 || feat_h < 1 || img_w < 1 || img_h < 1) return -100;
    if (static_cast<long long>(feat_w) * feat_h * per_loc >= kMaxPriors) return -200;
    const float step_w = param->step_w > 0.f ? param->step_w : static_cast<float>(img_w) / static_cast<float>(feat_w);
    const float step_h = param->step_h > 0.f ? param->step_h : static_cast<float>(img_h) / static_cast<float>(feat_h);
    return priorbox_forward(output, *param, per_loc, feat_w, feat_h, static_cast<float>(img_w), static_cast<float>(img_h),
                            step_w, step_h, as_stream(stream));
}

int fcuda_ssd_decode(float* boxes, const float* loc, const float* priors, int num_priors, int batch, void* stream) {
    if (!boxes || !loc || !priors || num_priors < 1 || batch < 1) return -100;
    if (num_priors >= kMaxPriors) return -200;
    return ssd_decode(boxes, loc, priors, num_priors, batch, as_stream(stream));
}

int fcuda_detection_output_workspace_size(int num_priors, int num_classes, int nms_top_k, int batch, size_t* floats) {
    if (!floats) return -100;
    const int rc = detection_limits(num_priors, num_classes, nms_top_k, batch);
    if (rc) return rc;
    *floats = detection_output_workspace(num_priors, num_classes, nms_top_k, batch);
    return 0;
}

int fcuda_detection_output_forward(float* output, const float* loc, const float* conf, const float* priors, int num_priors,
                                   int num_classes, float conf_threshold, float nms_threshold, int nms_top_k, int keep_top_k,
                                   float* workspace, int batch, void* stream) {
    const int rc = detection_limits(num_priors, num_classes, nms_top_k, batch);
    if (rc) return rc;
    if (keep_top_k < 1 || keep_top_k > 1024 || isnan(nms_threshold)) return -200;
    if (!output || !loc || !conf || !priors || !workspace || (reinterpret_cast<uintptr_t>(workspace) & 7)) return -100;
    return detection_output(output, loc, conf, priors, num_priors, num_classes, conf_threshold, nms_threshold, nms_top_k,
                            keep_top_k, workspace, batch, as_stream(stream));
}

static bool yolo_inputs_ok(const float* const* inputs, int scales) {
    if (!inputs) return false;
    for (int b = 0; b < scales; ++b)
        if (!inputs[b]) return false;
    return true;
}

int fcuda_yolo_decode(float* scores, int* classes, float* boxes, const float* const* inputs, const FcudaYoloParam* param,
                      int batch, void* stream) {
    int slots = 0;
    const int rc = yolo_limits(param, batch, &slots);
    if (rc) return rc;
    if (!scores || !classes || !boxes || !yolo_inputs_ok(inputs, param->num_scales)) return -100;
    return yolo_decode(scores, classes, boxes, inputs, *param, batch, as_stream(stream));
}

int fcuda_yolo_detection_workspace_size(const FcudaYoloParam* param, int batch, size_t* floats) {
    if (!floats) return -100;
    int slots = 0;
    const int rc = yolo_limits(param, batch, &slots);
    if (rc) return rc;
    *floats = yolo_detection_workspace(slots, batch);
    return 0;
}

int fcuda_yolo_detection_forward(float* output, const float* const* inputs, const FcudaYoloParam* param, float* workspace,
                                 int batch, void* stream) {
    int slots = 0;
    const int rc = yolo_limits(param, batch, &slots);
    if (rc) return rc;
    if (!output || !workspace || (reinterpret_cast<uintptr_t>(workspace) & 15) || !yolo_inputs_ok(inputs, param->num_scales))
        return -100;
    return yolo_detection(output, inputs, *param, workspace, batch, as_stream(stream));
}

static int proposal_limits(const FcudaProposalParam* p, int feat_h, int feat_w, int batch) {
    if (!p) return -100;
    if (p->feat_stride < 1 || p->base_size < 1 || p->pre_nms_topN < 1 || p->pre_nms_topN > 8192 || p->after_nms_topN < 1 ||
        p->after_nms_topN > 8192 || isnan(p->nms_thresh))
        return -200;
    if (batch < 1 || feat_h < 1 || feat_w < 1) return -100;
    if (batch > 65535 || feat_h >= kMaxPriors || feat_w >= kMaxPriors ||
        static_cast<long long>(FCUDA_PROPOSAL_ANCHORS) * feat_h * feat_w >= kMaxPriors)
        return -200;
    return 0;
}

int fcuda_proposal_anchors(const FcudaProposalParam* param, float* table) {
    const int rc = proposal_limits(param, 1, 1, 1);
    if (rc) return rc;
    if (!table) return -100;
    proposal_anchors(*param, table);
    return 0;
}

int fcuda_proposal_decode(float* boxes, const float* score, const float* bbox, const float* im_info,
                          const FcudaProposalParam* param, int feat_h, int feat_w, int batch, void* stream) {
    const int rc = proposal_limits(param, feat_h, feat_w, batch);
    if (rc) return rc;
    if (!boxes || !score || !bbox || !im_info) return -100;
    return proposal_decode(boxes, score, bbox, im_info, *param, feat_h, feat_w, batch, as_stream(stream));
}

int fcuda_proposal_workspace_size(const FcudaProposalParam* param, int feat_h, int feat_w, int batch, size_t* floats) {
    if (!floats) return -100;
    const int rc = proposal_limits(param, feat_h, feat_w, batch);
    if (rc) return rc;
    *floats = proposal_workspace(*param, feat_h, feat_w, batch);
    return 0;
}

int fcuda_proposal_forward(float* rois, float* scores, const float* score, const float* bbox, const float* im_info,
                           const FcudaProposalParam* param, int feat_h, int feat_w, float* workspace, int batch,
                           void* stream) {
    const int rc = proposal_limits(param, feat_h, feat_w, batch);
    if (rc) return rc;
    if (!rois || !score || !bbox || !im_info || !workspace || (reinterpret_cast<uintptr_t>(workspace) & 15)) return -100;
    return proposal_forward(rois, scores, score, bbox, im_info, *param, feat_h, feat_w, workspace, batch, as_stream(stream));
}

int fcuda_roi_pooling_forward(float* output, const float* input, const float* rois, int channels, int height, int width,
                              int num_rois, int pooled_h, int pooled_w, float spatial_scale, int batch, void* stream) {
    if (pooled_h < 1 || pooled_w < 1 || !isfinite(spatial_scale) || !(spatial_scale > 0.f)) return -200;
    if (!output || !input || !rois || channels < 1 || height < 1 || width < 1 || num_rois < 1 || batch < 1) return -100;
    return roi_pooling_forward(output, input, rois, channels, height, width, num_rois, pooled_h, pooled_w, spatial_scale,
                               batch, as_stream(stream));
}

int fcuda_psroi_pooling_forward(float* output, const float* input, const float* rois, int channels, int height,
                                int width, int num_rois, int pooled_h, int pooled_w, int output_dim, float spatial_scale,
                                int batch, void* stream) {
    if (pooled_h < 1 || pooled_w < 1 || output_dim < 1 || !isfinite(spatial_scale) || !(spatial_scale > 0.f) ||
        static_cast<long long>(output_dim) * pooled_h * pooled_w != channels)
        return -200;
    if (!output || !input || !rois || channels < 1 || height < 1 || width < 1 || num_rois < 1 || batch < 1) return -100;
    return psroi_pooling_forward(output, input, rois, channels, height, width, num_rois, pooled_h, pooled_w, output_dim,
                                 spatial_scale, batch, as_stream(stream));
}

static const long long kRouteMaxPositions = 1ll << 31;  // positions of the concatenated axis fit an int

int fcuda_route_forward(const FcudaRoute* route, int batch, void* stream) {
    if (!route) return -100;
    const FcudaRoute& r = *route;
    if (r.num_src < 1 || r.num_src > FCUDA_ROUTE_MAX || r.num_dst < 1 || r.num_dst > FCUDA_ROUTE_MAX) return -200;
    if (batch < 1 || r.outer < 1 || r.inner < 1 || r.dst_begin < 0) return -100;
    RouteGeom g;
    memset(&g, 0, sizeof(g));
    long long mid = 0, span = 0;
    for (int k = 0; k < r.num_src; ++k) {
        if (!r.src[k] || r.src_extent[k] < 1) return -100;
        g.src[k] = r.src[k];
        g.src_begin[k] = static_cast<int>(mid);
        mid += r.src_extent[k];
        if (mid >= kRouteMaxPositions) return -200;
    }
    for (int k = 0; k < r.num_dst; ++k) {
        if (!r.dst[k] || r.dst_extent[k] < 1) return -100;
        g.dst[k] = r.dst[k];
        g.dst_begin[k] = static_cast<int>(span);
        span += r.dst_extent[k];
        if (span >= kRouteMaxPositions) return -200;
    }
    g.src_begin[r.num_src] = static_cast<int>(mid);
    g.dst_begin[r.num_dst] = static_cast<int>(span);
    if (r.dst_begin + span > mid) return -100;
    if (r.group < 1 || mid % r.group != 0) return -200;
    if (static_cast<long long>(r.outer) * r.inner * span >= (1ll << 31)) return -200;
    g.num_src = r.num_src;
    g.num_dst = r.num_dst;
    g.first = r.dst_begin;
    g.g = r.reverse ? static_cast<int>(mid / r.group) : r.group;
    g.cpg = static_cast<int>(mid / g.g);
    g.outer = r.outer;
    g.inner = r.inner;
    return route_forward(g, batch, as_stream(stream));
}

int fcuda_slice_plan(int rank, int axis, const int* shape, const int* slices, int count, int* storage_axis, int* sizes) {
    if (!shape || !slices || !storage_axis || !sizes || count < 1 || rank < 1 || rank > 3) return -100;
    for (int k = 0; k < 3; ++k)
        if (shape[k] < 1) return -100;
    const int a = axis < 0 ? axis + rank : axis;
    if (a < 0 || a >= rank) return -200;
    const int sa = a + 3 - rank;
    const long long extent = shape[sa];
    long long taken = 0;
    for (int i = 0; i < count; ++i) {
        const long long n = slices[i] == -233 ? (extent - taken) / (count - i) : slices[i];
        if (n < 1 || taken + n > extent) return -200;
        sizes[i] = static_cast<int>(n);
        taken += n;
    }
    *storage_axis = sa;
    return 0;
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
