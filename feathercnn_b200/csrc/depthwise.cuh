#pragma once
#include <cuda_runtime.h>
namespace fcuda {
struct DwGeom {
    int C, H, W, KH, KW, OH, OW, stride_h, stride_w, pad_top, pad_left;
};
// out[n][c] = act(in[n][c] (*) w[c] + bias[c]); w is (C, KH, KW); act: 0 none, 1 ReLU, 2 Clip to [lo, hi].
int depthwise_forward(const float* in, const float* w, const float* bias, float* out, const DwGeom& g, int act, float lo,
                      float hi, int batch, cudaStream_t s);
}  // namespace fcuda
