// Implicit-GEMM convolution on Hopper warpgroup MMA (see conv_igemm.cu).
#pragma once
#include <cuda_runtime.h>

namespace fcuda {

struct IgemmProblem {
    const float* input;   // (N, IC, H, W) fp32 NCHW
    const float* w_hi;    // packed filters [OC][Kf], k = tap*IC + ic, TF32-exact plane
    const float* w_lo;    // fp32 remainder plane (planes == 2) or null
    const float* bias;    // OC floats or null
    float* output;        // (N, OC, OH, OW)
    int N, IC, H, W, OC, OH, OW;
    int KH, KW, pad_top, pad_left, stride_h, stride_w;
    int planes;           // 1 = TF32, 2 = 3xTF32, 3 = BF16x3 (w_hi / w_lo then hold the two bf16 planes)
    int relu;
    const float* residual;  // optional (N, OC, OH, OW) tensor added before the activation (fused Eltwise SUM), or null
    // Extensions beyond the reference (it rejects both: conv_layer.h:43-47, avx/booster.cpp:304-308); 0 = default.
    int dil_h, dil_w;       // dilation (0 or 1 = dense taps)
    int in_c_total;         // channels per image of the INPUT tensor when `input` addresses a channel slice of it
    int out_c_total;        // same for output / residual (grouped convolution = one launch per group on slices)
    int pool;               // fuse a following 2x2 / stride-2 max pooling (pad 0): `output` is (N, OC, (OH+1)/2, (OW+1)/2)
};

// KH*KW <= 63 and, unless IC % 32 == 0, KH*KW*IC <= 8192 (shared-memory k-table).
bool conv_igemm_supported(int IC, int KH, int KW);
// Floats of the packed filter buffer ([OC][Kf] per plane, Kf = KH*KW*IC rounded up to 4).
size_t conv_igemm_packed_floats(int OC, int IC, int taps, int planes);
// raw (OC, IC, KH, KW) -> [OC][Kf] hi (+ lo) planes.
// bf16x3 != 0: w_hi / w_lo receive the two bf16 planes q1 = RN(w), q2 = RN(w - q1), rows of Kf8 = K rounded up to 8
// (they fit the float planes sized above).
int conv_igemm_pack_weights(const float* w, float* w_hi, float* w_lo, int OC, int IC, int taps, cudaStream_t s,
                            int bf16x3 = 0);
// True when the launch can apply a fused 2x2 / stride-2 max pooling (the 3x3 stride-1 slab kernel without a residual).
bool conv_igemm_can_pool(const IgemmProblem& p);
// Output patch (R x C pixels) and shared-memory halo box (Rb x Cb) of the halo kernel conv_igemm_forward uses for
// stride-1, dense layers with IC % 32 == 0 and W % 4 == 0 (switch igemm_halo); false when the layer keeps the
// gathering kernel.  Reads IC, OC, H, W, OH, OW, KH, KW, strides, dilation, planes and the input address.
struct HaloGeom { int R, C, Rb, Cb; };
bool conv_igemm_halo_geometry(const IgemmProblem& p, HaloGeom* g);
// Tile (R x C pixels, R * C = 128 or 256) and box of the pre-split halo kernel conv_igemm_forward uses in BF16x3 mode
// (switch igemm_presplit) on a layer that takes the halo kernel; false when the layer keeps the halo kernel.
bool conv_igemm_presplit_geometry(const IgemmProblem& p, HaloGeom* g);
int conv_igemm_forward(const IgemmProblem& p, cudaStream_t stream);

}  // namespace fcuda
