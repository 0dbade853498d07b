// ncnn's BinaryOp: out = op(a, b) over NCHW fp32 blobs, with a scalar or a broadcast operand (fcuda_binary_op_forward).
//
// Two kernels, each instantiated per op so the loop body is one operation:
//   same shape (or a scalar b): a flat pass over n floats, float4 loads and stores where all pointers are 16-byte
//     aligned, then a scalar tail;
//   broadcast: one thread per kBinaryVec consecutive outputs of a row.  It splits its item into (n, c, y, x0) once, with
//     32-bit divisions while the item fits in 32 bits, and reads each operand through its strides (0 on the axes it
//     broadcasts).  Planes are part of the 1-D item index in gridDim.x, so any number of (n, c) planes fits the grid.
// The same-shape ADD never reaches this file: it is Eltwise SUM and runs on add_relu (layers.cu).
#include "fcuda.h"

#include "binary_op.cuh"
#include "common.cuh"

#include <stdint.h>

namespace fcuda {

constexpr int kBinaryThreads = 256;
constexpr int kBinaryVec = 4;  // consecutive outputs of one row per thread (broadcast kernel)

template <int OP>
__device__ __forceinline__ float binary_apply(float a, float b) {
    if constexpr (OP == FCUDA_BINARY_ADD) return a + b;
    else if constexpr (OP == FCUDA_BINARY_SUB) return a - b;
    else if constexpr (OP == FCUDA_BINARY_MUL) return a * b;
    else if constexpr (OP == FCUDA_BINARY_DIV) return a / b;  // IEEE division: the build has no fast-math
    else if constexpr (OP == FCUDA_BINARY_MAX) return fmaxf(a, b);
    else if constexpr (OP == FCUDA_BINARY_MIN) return fminf(a, b);
    else if constexpr (OP == FCUDA_BINARY_POW) return powf(a, b);
    else if constexpr (OP == FCUDA_BINARY_RSUB) return b - a;
    else if constexpr (OP == FCUDA_BINARY_RDIV) return b / a;
    else if constexpr (OP == FCUDA_BINARY_RPOW) return powf(b, a);
    else if constexpr (OP == FCUDA_BINARY_ATAN2) return atan2f(a, b);
    else return atan2f(b, a);  // FCUDA_BINARY_RATAN2
}

template <int OP>
__device__ __forceinline__ float binary_out(float a, float b, int relu) {
    const float r = binary_apply<OP>(a, b);
    return relu ? fmaxf(r, 0.f) : r;  // the Eltwise ReLU (add_relu_kernel): NaN becomes 0
}

// Plain loads: out may be a or b.
template <int OP>
__global__ void __launch_bounds__(kBinaryThreads)
binary_same_kernel(float* out, const float* a, const float* b, float bs, size_t n, int relu) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(out)) &
                      15) == 0;
    const size_t nv = vec ? n >> 2 : 0;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
        const float4 x = reinterpret_cast<const float4*>(a)[i];
        const float4 y = b ? reinterpret_cast<const float4*>(b)[i] : make_float4(bs, bs, bs, bs);
        reinterpret_cast<float4*>(out)[i] = make_float4(binary_out<OP>(x.x, y.x, relu), binary_out<OP>(x.y, y.y, relu),
                                                        binary_out<OP>(x.z, y.z, relu), binary_out<OP>(x.w, y.w, relu));
    }
    for (size_t i = (nv << 2) + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = binary_out<OP>(a[i], b ? b[i] : bs, relu);
}

__device__ __forceinline__ unsigned long long div_u(unsigned long long x, unsigned d) {
    return (x >> 32) ? x / d : static_cast<unsigned>(x) / d;
}

// VEC: W % 4 == 0 and out 16-byte aligned, so a thread's outputs are one float4 store.
template <int OP, bool VEC>
__global__ void __launch_bounds__(kBinaryThreads)
binary_broadcast_kernel(float* out, BinaryOperand a, BinaryOperand b, int C, int H, int W, int groups,
                        unsigned long long items, int relu) {
    const unsigned long long item = static_cast<unsigned long long>(blockIdx.x) * kBinaryThreads + threadIdx.x;
    if (item >= items) return;
    const unsigned long long row = div_u(item, static_cast<unsigned>(groups));  // plane * H + y
    const int x0 = static_cast<int>(item - row * groups) * kBinaryVec;
    const unsigned long long plane = div_u(row, static_cast<unsigned>(H));
    const int y = static_cast<int>(row - plane * H);
    const long long n = static_cast<long long>(div_u(plane, static_cast<unsigned>(C)));
    const int c = static_cast<int>(plane - static_cast<unsigned long long>(n) * C);
    const float* pa = a.p + n * a.sn + c * a.sc + y * a.sh;
    const float* pb = b.p + n * b.sn + c * b.sc + y * b.sh;
    float r[kBinaryVec];
#pragma unroll
    for (int k = 0; k < kBinaryVec; ++k) {
        const int x = min(x0 + k, W - 1);  // past the row's end: a valid element, computed and not stored
        r[k] = binary_out<OP>(pa[x * a.sw], pb[x * b.sw], relu);
    }
    float* dst = out + row * W + x0;
    if constexpr (VEC) {
        *reinterpret_cast<float4*>(dst) = make_float4(r[0], r[1], r[2], r[3]);
    } else {
#pragma unroll
        for (int k = 0; k < kBinaryVec; ++k)
            if (x0 + k < W) dst[k] = r[k];
    }
}

using SameKernel = void (*)(float*, const float*, const float*, float, size_t, int);
using BroadcastKernel = void (*)(float*, BinaryOperand, BinaryOperand, int, int, int, int, unsigned long long, int);

template <int... OPS>
struct BinaryTable {
    static constexpr SameKernel same[] = {binary_same_kernel<OPS>...};
    static constexpr BroadcastKernel row[] = {binary_broadcast_kernel<OPS, false>...};
    static constexpr BroadcastKernel row4[] = {binary_broadcast_kernel<OPS, true>...};
};
using Ops = BinaryTable<0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11>;

int binary_op_same(float* out, const float* a, const float* b, float b_scalar, size_t n, int op, int relu,
                   cudaStream_t s) {
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0, (b ? 12.0 : 8.0) * n);
    size_t blocks = ceil_div_sz(n / 4 + 1, kBinaryThreads);
    const size_t cap = static_cast<size_t>(sm_count()) * 32;
    if (blocks > cap) blocks = cap;
    Ops::same[op]<<<static_cast<unsigned>(blocks), kBinaryThreads, 0, s>>>(out, a, b, b_scalar, n, relu);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

// The bytes an operand must move: its distinct elements, once.
static double operand_floats(const BinaryOperand& o, int C, int H, int W, int batch) {
    return static_cast<double>(batch) * (o.sc ? C : 1) * (o.sh ? H : 1) * (o.sw ? W : 1);
}

int binary_op_broadcast(float* out, const BinaryOperand& a, const BinaryOperand& b, int C, int H, int W, int op,
                        int relu, int batch, cudaStream_t s) {
    const double out_n = static_cast<double>(batch) * C * H * W;
    const int prof = prof_begin(s, PROF_ELEMENTWISE, 0, 0,
                                4.0 * (out_n + operand_floats(a, C, H, W, batch) + operand_floats(b, C, H, W, batch)));
    const int groups = ceil_div(W, kBinaryVec);
    const unsigned long long items = static_cast<unsigned long long>(batch) * C * H * groups;
    const unsigned blocks = static_cast<unsigned>((items + kBinaryThreads - 1) / kBinaryThreads);
    const bool vec = W % kBinaryVec == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    (vec ? Ops::row4 : Ops::row)[op]<<<blocks, kBinaryThreads, 0, s>>>(out, a, b, C, H, W, groups, items, relu);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
