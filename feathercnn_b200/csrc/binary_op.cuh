#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
namespace fcuda {

// ncnn's BinaryOp after validation (fcuda_binary_op_forward): out = op(a, b), then fmaxf(., 0) with `relu`.  `op` is
// 0..11 in ncnn's numbering (include/fcuda.h).  Neither allocates nor synchronises.

// Same shape, n floats each; `b` null stands for the scalar `b_scalar`.  out == a or out == b is allowed.
int binary_op_same(float* out, const float* a, const float* b, float b_scalar, size_t n, int op, int relu,
                   cudaStream_t s);

// An operand of the broadcast form: its element strides along n, c, h, w of the output, 0 on the axes it broadcasts.
struct BinaryOperand {
    const float* p;
    long long sn, sc, sh, sw;
};
// Output (batch, C, H, W), H * W < 2^31; out may be an operand that broadcasts on no axis.
int binary_op_broadcast(float* out, const BinaryOperand& a, const BinaryOperand& b, int C, int H, int W, int op,
                        int relu, int batch, cudaStream_t s);
}  // namespace fcuda
