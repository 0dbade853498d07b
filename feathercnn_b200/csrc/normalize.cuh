#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
namespace fcuda {

// ncnn's Normalize after validation (fcuda_normalize_forward): y = (x * a) * scale[shared ? 0 : c] with
// a = normalize_factor(sum of x^2 over the reduction set).  across_spatial 0: the C values of one pixel (one launch);
// across_spatial 1: the whole image (across_channel 1) or one channel plane (across_channel 0), two launches through
// `workspace` (normalize_workspace_floats of them).
struct NormalizeGeom {
    int channels;
    size_t plane;
    int batch;
    int across_spatial, across_channel;
    int shared;
    float eps;
    int eps_mode;
};
size_t normalize_workspace_floats(int across_spatial, int across_channel, int channels, size_t plane, int batch);
int normalize_forward(const float* in, float* out, const float* scale, const NormalizeGeom& g, float* workspace,
                      cudaStream_t s);
}  // namespace fcuda
