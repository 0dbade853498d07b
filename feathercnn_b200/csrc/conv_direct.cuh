#pragma once
#include "common.cuh"
#include "pack.cuh"
namespace fcuda {
// out[n][oc][pix] = act(sum_k w[oc][k] * im2col(in[n])[k][pix] + bias[oc]), fp32 FMA on CUDA cores; reads e.bias and
// e.act / lo / hi.
int conv_direct(const float* in, const float* w, float* out, const PackGeom& g, int OC, const ConvEpilogue& e, int batch,
                cudaStream_t s);
}  // namespace fcuda
