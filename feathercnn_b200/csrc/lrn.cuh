#pragma once
#include <cuda_runtime.h>
namespace fcuda {

// ncnn's LRN after validation (fcuda_lrn_forward): region 0 across channels, 1 within each channel plane; local_size odd
// and >= 1; out of place.  fcuda.h states the arithmetic and the summation order.
struct LrnGeom {
    int channels, h, w, batch;
    int region, local_size;
    float alpha, beta, bias;
};
int lrn_forward(const float* in, float* out, const LrnGeom& g, cudaStream_t s);
}  // namespace fcuda
