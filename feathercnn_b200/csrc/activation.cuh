#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
namespace fcuda {

// The logistic sigmoid, 1 / (1 + expf(-t)), with the add and the division rounded once each (IEEE division).  Shared by
// the Sigmoid / Swish layers and the YOLO decode (detection.cu), so both give the same bits.
__device__ __forceinline__ float sigm(float t) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-t))); }

// ncnn's Sigmoid / TanH / Swish / HardSigmoid / HardSwish over n floats after validation (fcuda_activation_forward).
// `type` is an FcudaActivationType; alpha, beta, lower, upper are used by the hard types only.  out == in is allowed.
// Neither allocates nor synchronises.
int activation(float* out, const float* in, size_t n, int type, float alpha, float beta, float lower, float upper,
               cudaStream_t s);
}  // namespace fcuda
