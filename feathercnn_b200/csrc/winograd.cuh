// Winograd transform launchers (see winograd.cu).
#pragma once
#include <cuda_runtime.h>

namespace fcuda {

struct WinoGeom {
    int C_in, C_out;
    int H, W;          // unpadded input
    int OH, OW;        // output
    int pad_top, pad_left;
    int tilesX, tilesY;  // ceil(OW / out_tile), ceil(OH / out_tile) — (Wp+3)/6, (Hp+3)/6 in the reference
};

// tile = 8 (F(6,3)) or 4 (F(2,3)).  U_lo may be null (plain TF32 mode); V is always one plain-fp32 plane.
int wino_filter_transform(int tile, const float* w, float* U_hi, float* U_lo, int OC, int IC, cudaStream_t s);
// Transforms tile-rows [R0, R1) (a tile-row = one row of tiles of one image; R = img * tilesY + ty).
int wino_input_transform(int tile, const float* in, float* V, const WinoGeom& g, int R0, int R1, cudaStream_t s);
// act: 0 none, 1 ReLU, 2 Clip to [lo, hi].  pool != 0: a following 2x2 / stride-2 max pooling is applied in registers; `out` is the pooled (C_out, (OH+1)/2, (OW+1)/2) blob.
int wino_output_transform(int tile, const float* M, float* out, const float* bias, const WinoGeom& g, int R0, int R1,
                          int act, float lo, float hi, int pool, cudaStream_t s);

}  // namespace fcuda
