#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
namespace fcuda {

// A plane padding after validation (fcuda_padding_forward / fcuda_instance_norm_forward): type 0 constant, 1
// replicate, 2 reflect (edge excluded); every pad >= 0 and, for reflect, below the dimension it pads.
struct PlanePad {
    int top, bottom, left, right;
    int type;
    float value;
};

// ncnn's InstanceNorm after validation: per (n, c) plane of h * w floats, y = fmaf(x, a, b) from the plane's mean and
// biased variance (two launches through `workspace`, instance_norm_workspace_floats of them), then an optional ReLU
// and an optional padding of the output plane (`pad` NULL: none; output != input when set).
size_t instance_norm_workspace_floats(int channels, size_t plane, int batch);
int instance_norm_forward(const float* in, float* out, int channels, int h, int w, const float* gamma,
                          const float* beta, float eps, int relu, const PlanePad* pad, float* workspace, int batch,
                          cudaStream_t s);
// Padding alone: a copy of each plane through the same index function (out != in unless every pad is 0).
int padding_forward(const float* in, float* out, int channels, int h, int w, const PlanePad& pad, int batch,
                    cudaStream_t s);
}  // namespace fcuda
