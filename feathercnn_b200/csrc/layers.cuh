#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
namespace fcuda {
struct PoolGeom {
    int H, W, OH, OW, KH, KW, stride_h, stride_w, pad_left, pad_right, pad_top, pad_bottom, type;
};
int pooling_forward(const float* in, float* out, const PoolGeom& g, int channels, int batch, cudaStream_t s);
// y = act(((mul*x + add) * mul2) + add2) per channel; null pointers skip the term.
int channel_affine(const float* in, float* out, int channels, size_t hw, const float* mul, const float* add,
                   const float* mul2, const float* add2, int relu, int batch, cudaStream_t s);
int add_relu(const float* a, const float* b, float* out, size_t n, int relu, cudaStream_t s);
// op 0 = a*b, 1 = ca*a + cb*b, 2 = max(a, b); then optional ReLU (ncnn Eltwise semantics)
int eltwise(const float* a, const float* b, float* out, size_t n, int op, float ca, float cb, int relu, cudaStream_t s);
int scale_relu(const float* in, float* out, size_t n, float scale, int relu, cudaStream_t s);
// y = min(max(x, lo), hi) (NaN -> lo); in place allowed.
int clip(const float* in, float* out, size_t n, float lo, float hi, cudaStream_t s);
// y = x < 0 ? x * slope[c] : x over (batch, channels, plane); shared != 0: slope[0] for every channel.  In place allowed.
int prelu(const float* in, float* out, const float* slope, int channels, size_t plane, int shared, int batch,
          cudaStream_t s);
int softmax_forward(const float* in, float* out, size_t n_per_image, int batch, cudaStream_t s);
int copy_channels(const float* src, float* dst, size_t per_image, size_t dst_image, size_t dst_offset, int batch,
                  cudaStream_t s);
// out[r][j] = act(bias[j] + sum_s part[s][r][j]); fixed summation order (deterministic split-K reduction).
int fc_reduce(float* out, const float* part, const float* bias, int splits, int row_len, int rows, int relu,
              cudaStream_t s);
// out[r][j] = row[j] (or 0 when row is null) for r < rows.
int fill_rows(float* out, const float* row, int row_len, int rows, cudaStream_t s);
}  // namespace fcuda
