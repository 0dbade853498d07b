#pragma once
#include <cuda_runtime.h>
namespace fcuda {
// Sub-pixel scatter of a deconvolution computed as one stride-1 convolution P with channels ordered
// (group, r_y, r_x, oc_in_group):  out[n][oc][oy][ox] = act(P[n][(g, Y % s_h, X % s_w, oc)][Y / s_h][X / s_w] + bias[oc]),
// Y = oy + pad_top, X = ox + pad_left, and 0 in place of P where Y / s_h >= Hc or X / s_w >= Wc.
struct DeconvScatterGeom {
    int OC, group, stride_h, stride_w, Hc, Wc, OH, OW, pad_top, pad_left;
};
// With `add` (the PixelShuffle tail), the scatter then adds add.base[n][oc][nearest_coord(oy, H, scale_h)]
// [nearest_coord(ox, W, scale_w)], one fp32 add, as a nearest Interp of base followed by an Eltwise SUM.  `kind` is
// the profiling kind the launch is counted under.
struct ScatterAddend {
    const float* base;
    int H, W;
    float scale_h, scale_w;
};
int deconv_scatter(const float* P, const float* bias, float* out, const DeconvScatterGeom& g, int relu,
                   const ScatterAddend* add, int kind, int batch, cudaStream_t s);

// Depthwise deconvolution (one filter per channel, w is (C, KH, KW)): every output gathers its taps in ascending
// (ky, kx) order with fp32 FMAs, starting from the bias; stride > 1 and dilation > 1 never share a direction.
struct DeconvDwGeom {
    int C, H, W, KH, KW, stride_h, stride_w, dil_h, dil_w, pad_top, pad_left, OH, OW;
};
int deconv_depthwise(const float* in, const float* w, const float* bias, float* out, const DeconvDwGeom& g, int relu,
                     int batch, cudaStream_t s);
}  // namespace fcuda
