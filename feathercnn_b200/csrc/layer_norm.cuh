#pragma once
#include <cuda_runtime.h>
namespace fcuda {
// fcuda_layer_norm_forward after validation: `rows` rows of n floats, gamma / beta both set or both NULL.  out == in is
// allowed.  Neither allocates nor synchronises.
int layer_norm(float* out, const float* in, int n, long long rows, const float* gamma, const float* beta, float eps,
               cudaStream_t s);
}  // namespace fcuda
