// Implicit-GEMM convolution on Hopper warpgroup MMA (see conv_igemm.cu).
#pragma once
#include "common.cuh"

namespace fcuda {

struct IgemmProblem {
    const float* input;   // (N, IC, H, W) fp32 NCHW
    const float* w_hi;    // packed filters [OC][Kf], k = tap*IC + ic, TF32-exact plane
    const float* w_lo;    // fp32 remainder plane (planes == 2) or null
    float* output;        // (N, OC, OH, OW)
    int N, IC, H, W, OC, OH, OW;
    int KH, KW, pad_top, pad_left, stride_h, stride_w;
    int planes;           // 1 = TF32, 2 = 3xTF32, 3 = BF16x3 (w_hi then holds both pre-tiled bf16 planes)
    ConvEpilogue epi;     // every field is read; with epi.pool `output` is (N, OC, (OH+1)/2, (OW+1)/2)
    // Extensions beyond the reference (it rejects both: conv_layer.h:43-47, avx/booster.cpp:304-308); 0 = default.
    int dil_h, dil_w;       // dilation (0 or 1 = dense taps)
    int in_c_total;         // channels per image of the INPUT tensor when `input` addresses a channel slice of it
    int out_c_total;        // same for output / residual (grouped convolution = one launch per group on slices)
};

// KH*KW <= 63 and, unless IC % 32 == 0, KH*KW*IC <= 6144 (shared-memory k-table).
bool conv_igemm_supported(int IC, int KH, int KW);
// Floats of the packed filter buffer: [OC][Kf] per plane (Kf = KH*KW*IC rounded up to 4), or with planes >= 2 at
// least the pre-tiled BF16x3 planes.
size_t conv_igemm_packed_floats(int OC, int IC, int taps, int planes);
// raw (OC, IC, KH, KW) -> [OC][Kf] hi (+ lo) planes.
// bf16x3 != 0: w_hi receives both bf16 planes q1 = RN(w), q2 = RN(w - q1), pre-tiled per (32-wide k-block, N tile) in
// the un-swizzled core-matrix order of wgmma, so that one bulk copy fetches a filter stage; w_lo is not written.
int conv_igemm_pack_weights(const float* w, float* w_hi, float* w_lo, int OC, int IC, int taps, cudaStream_t s,
                            int bf16x3 = 0);
// True when the launch can apply a fused 2x2 / stride-2 max pooling: 3x3, stride 1, no dilation, IC % 32 == 0, pads
// <= 2, W % 4 == 0, a 16-byte aligned (or not yet known) input and no residual.
bool conv_igemm_can_pool(const IgemmProblem& p);
// Output patch (R x C pixels) and shared-memory halo box (Rb x Cb) of the halo kernel conv_igemm_forward uses for
// stride-1, dense layers with IC % 32 == 0 and W % 4 == 0 (switch igemm_halo); false when the layer keeps the
// gathering kernel.  Reads IC, OC, H, W, OH, OW, KH, KW, strides, dilation, planes and the input address.
struct HaloGeom { int R, C, Rb, Cb; };
bool conv_igemm_halo_geometry(const IgemmProblem& p, HaloGeom* g);
// Tile (R x C pixels, R * C = 128) and box of the pre-split halo kernel conv_igemm_forward uses in BF16x3 mode
// (switch igemm_presplit) on a layer that takes the halo kernel; false when the layer keeps the halo kernel.
bool conv_igemm_presplit_geometry(const IgemmProblem& p, HaloGeom* g);
// Tile (28 x 16 pixels with a 64-channel N tile, 28 x 8 with a 128-channel one) and box of the wide pre-split kernel
// (switch igemm_wide) on a layer that takes the pre-split kernel; false when the layer keeps the pre-split kernel.
bool conv_igemm_wide_geometry(const IgemmProblem& p, HaloGeom* g);
// True when the layer takes the persistent stem kernel (switch igemm_stem): BF16x3 mode, IC % 32 != 0, KH*KW*IC <= 256,
// OC <= 128, no residual, pooling or dilation.  Reads planes, IC, OC, H, W, OH, OW, KH, KW, dilation and epi.
bool conv_igemm_stem_supported(const IgemmProblem& p);
int conv_igemm_forward(const IgemmProblem& p, cudaStream_t stream);

}  // namespace fcuda
