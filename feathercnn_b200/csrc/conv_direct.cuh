#pragma once
#include "pack.cuh"
namespace fcuda {
// out[n][oc][pix] = act(sum_k w[oc][k] * im2col(in[n])[k][pix] + bias[oc]), fp32 FMA on CUDA cores; act: 0 none,
// 1 ReLU, 2 Clip to [lo, hi].
int conv_direct(const float* in, const float* w, const float* bias, float* out, const PackGeom& g, int OC, int act,
                float lo, float hi, int batch, cudaStream_t s);
}  // namespace fcuda
