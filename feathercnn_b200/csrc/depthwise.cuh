#pragma once
#include "common.cuh"
namespace fcuda {
struct DwGeom {
    int C, H, W, KH, KW, OH, OW, stride_h, stride_w, pad_top, pad_left;
    int dil_h, dil_w;  // tap spacing; 0 means 1
};
// out[n][c] = act(in[n][c] (*) w[c] + bias[c]); w is (C, KH, KW); reads e.bias and e.act / lo / hi.
int depthwise_forward(const float* in, const float* w, float* out, const DwGeom& g, const ConvEpilogue& e, int batch,
                      cudaStream_t s);
}  // namespace fcuda
