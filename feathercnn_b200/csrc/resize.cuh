#pragma once
#include <cuda_runtime.h>
namespace fcuda {
// ncnn Interp on `planes` = batch * C planes of H x W -> OH x OW.  mode 1 nearest: source index
// min((int)(d * scale), in - 1).  mode 2 bilinear: source coordinate (d + 0.5) * scale - 0.5 clamped at 0
// (align_corner = 0) or d * scale (align_corner = 1), neighbours i0 = (int)f and min(i0 + 1, in - 1).
// scale_h / scale_w are the fp32 ratios fcuda_interp_forward derives from the parameters.
struct InterpGeom {
    int H, W, OH, OW, mode, align_corner;
    float scale_h, scale_w;
};
int interp_forward(const float* in, float* out, const InterpGeom& g, long long planes, cudaStream_t s);

// ncnn's nearest index: min((int)(d * scale), in - 1) with the fp32 product.  Shared by Interp and the PixelShuffle
// tail that adds a nearest-upsampled blob (deconv.cu), so both read the same source element.
__device__ __forceinline__ int nearest_coord(int d, int in, float scale) {
    return min(static_cast<int>(__fmul_rn(static_cast<float>(d), scale)), in - 1);
}

// out[n][c][y][x] = in[n][c + coff][y + hoff][x + woff] for an out_c x out_h x out_w window of each image.
struct CropGeom {
    int C, H, W, coff, hoff, woff, OC, OH, OW;
};
int crop_forward(const float* in, float* out, const CropGeom& g, int batch, cudaStream_t s);
}  // namespace fcuda
