#pragma once
#include <cuda_runtime.h>
namespace fcuda {
// fcuda_attention_forward after validation: d one of 16, 32, ..., 128, heads * ceil(lq / 64) <= 65535.  Neither allocates
// nor synchronises.
int attention(float* o, const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, int batch,
              int heads, int d, int lq, int lk, float scale, cudaStream_t s);
}  // namespace fcuda
