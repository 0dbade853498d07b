// Winograd transform launchers (see winograd.cu).
#pragma once
#include "common.cuh"

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
// Reads e.bias, e.act / lo / hi and e.pool (the pooling is applied in registers).
int wino_output_transform(int tile, const float* M, float* out, const WinoGeom& g, int R0, int R1, const ConvEpilogue& e,
                          cudaStream_t s);

}  // namespace fcuda
