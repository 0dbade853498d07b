// Fused scaled dot-product attention for MultiHeadAttention (fcuda_attention_forward): the score tile lives in registers
// and never reaches global memory.
//
// One warpgroup per CTA owns 64 query rows of one (image, head).  Per key tile of 64:
//   1. all 128 threads stage K and V from fp32 global memory into shared memory as bf16 p1 / p2 planes (the BF16x3
//      split), in the un-swizzled K-major core-matrix layout wgmma reads: K as [key][d], V transposed to [d][key];
//   2. S = Q K^T: 3 d / 16 wgmma (p2 q1, p1 q2, p1 q1 per k-step of 16) with Q's fragments split once in registers;
//   3. the online softmax in fp32 on the accumulators (row max and sum over the 4 lanes of a row by xor shuffles);
//   4. O += P V: 12 wgmma with P's fragments split in registers straight from the accumulator layout.
// Each product is one commit group waited on once, so its wgmma run back to back.  The order of every operation is
// fixed by the tile walk, so the bits depend on neither the batch split nor the launch.
#include "fcuda.h"

#include "common.cuh"
#include "wgmma.cuh"

#include <math.h>
#include <stdint.h>

namespace fcuda {

constexpr int kAttnThreads = 128;
constexpr int kAttnBM = 64;  // queries per CTA
constexpr int kAttnBN = 64;  // keys per tile

template <int D>
constexpr int attn_smem_bytes() { return 4 * kAttnBN * D * 2; }  // K p1 / p2, V p1 / p2, bf16

template <int D>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_kernel(float* __restrict__ o, const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                 const float* __restrict__ v, int ldv, int heads, int lq, int lk, float scale) {
    constexpr int KS = D / 16;  // k-steps of S = Q K^T
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* k_hi = smem;
    uint8_t* k_lo = smem + kAttnBN * D * 2;
    uint8_t* v_hi = smem + 2 * kAttnBN * D * 2;
    uint8_t* v_lo = smem + 3 * kAttnBN * D * 2;

    const int b = blockIdx.x;
    const int h = blockIdx.y % heads;
    const int q0 = (blockIdx.y / heads) * kAttnBM;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const float* qb = q + static_cast<size_t>(b) * lq * ldq + h * D;
    const float* kb = k + static_cast<size_t>(b) * lk * ldk + h * D;
    const float* vb = v + static_cast<size_t>(b) * lk * ldv + h * D;
    const int r0 = q0 + 16 * warp + g, r1 = r0 + 8;

    // Q's A fragments (rows r0 / r1, columns 16 kk + 2c (+1) and + 8), split once: qa1 = p1, qa2 = p2
    uint32_t qa1[KS][4], qa2[KS][4];
#pragma unroll
    for (int kk = 0; kk < KS; ++kk)
#pragma unroll
        for (int f = 0; f < 4; ++f) {
            const int row = (f & 1) ? r1 : r0;
            const int col = 16 * kk + 2 * c + 8 * (f >> 1);
            float x0 = 0.f, x1 = 0.f;
            if (row < lq) {
                x0 = qb[static_cast<size_t>(row) * ldq + col];
                x1 = qb[static_cast<size_t>(row) * ldq + col + 1];
            }
            split_bf16x2(x0, x1, qa1[kk][f], qa2[kk][f]);
        }

    float oacc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) oacc[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    const uint32_t k_hi_a = ptx::smem_u32(k_hi), k_lo_a = ptx::smem_u32(k_lo);
    const uint32_t v_hi_a = ptx::smem_u32(v_hi), v_lo_a = ptx::smem_u32(v_lo);
    const int sr = lane & 7, sw = lane >> 3;  // staging: row of a core matrix, pair of columns in it
    const int tiles = (lk + kAttnBN - 1) / kAttnBN;

    for (int t = 0; t < tiles; ++t) {
        const int key0 = t * kAttnBN;
        __syncthreads();  // every warp's wgmma of the previous tile have completed (each waited) before smem is rewritten
        // K: core matrix (key group kg, d chunk dc) at kg * 16 D + dc * 128 bytes; lane -> (key kg 8 + sr, d dc 8 + 2 sw)
        for (int idx = warp; idx < D; idx += 4) {
            const int kg = idx / (D / 8), dc = idx % (D / 8);
            const int key = key0 + 8 * kg + sr, col = 8 * dc + 2 * sw;
            float x0 = 0.f, x1 = 0.f;
            if (key < lk) {
                x0 = kb[static_cast<size_t>(key) * ldk + col];
                x1 = kb[static_cast<size_t>(key) * ldk + col + 1];
            }
            uint32_t p1, p2;
            split_bf16x2(x0, x1, p1, p2);
            const int off = kg * 16 * D + dc * 128 + sr * 16 + sw * 4;
            *reinterpret_cast<uint32_t*>(k_hi + off) = p1;
            *reinterpret_cast<uint32_t*>(k_lo + off) = p2;
        }
        // V^T: core matrix (d group dg, key chunk kc) at dg * 1024 + kc * 128 bytes; lane -> (d dg 8 + sr, keys kc 8 + 2 sw, +1)
        for (int idx = warp; idx < D; idx += 4) {
            const int dg = idx / 8, kc = idx % 8;
            const int key = key0 + 8 * kc + 2 * sw, col = 8 * dg + sr;
            const float x0 = key < lk ? vb[static_cast<size_t>(key) * ldv + col] : 0.f;
            const float x1 = key + 1 < lk ? vb[static_cast<size_t>(key + 1) * ldv + col] : 0.f;
            uint32_t p1, p2;
            split_bf16x2(x0, x1, p1, p2);
            const int off = dg * 1024 + kc * 128 + sr * 16 + sw * 4;
            *reinterpret_cast<uint32_t*>(v_hi + off) = p1;
            *reinterpret_cast<uint32_t*>(v_lo + off) = p2;
        }
        ptx::fence_proxy_async_smem();
        __syncthreads();

        // S = Q K^T (64 x 64 per warpgroup)
        float sacc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) sacc[i] = 0.f;
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
            const uint64_t d1 = make_smem_desc_none(k_hi_a + 256 * kk, 128, 16 * D);
            const uint64_t d2 = make_smem_desc_none(k_lo_a + 256 * kk, 128, 16 * D);
            Wgmma<64, 0>::mma(sacc, qa2[kk], d1, 1u);  // p2 * q1
            Wgmma<64, 0>::mma(sacc, qa1[kk], d2, 1u);  // p1 * q2
            Wgmma<64, 0>::mma(sacc, qa1[kk], d1, 1u);  // p1 * q1
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();

        // online softmax: sacc[4j + i] is row (i >> 1 ? r1 : r0), key key0 + 8j + 2c + (i & 1)
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int key = key0 + 8 * j + 2 * c + (i & 1);
                const float s = key < lk ? __fmul_rn(sacc[4 * j + i], scale) : -INFINITY;
                sacc[4 * j + i] = s;
                if (i >> 1) mx1 = fmaxf(mx1, s);
                else mx0 = fmaxf(mx0, s);
            }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
        }
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);  // finite: every tile holds at least one key
        const float al0 = expf(__fsub_rn(m0, mn0)), al1 = expf(__fsub_rn(m1, mn1));  // 0 on the first tile
        m0 = mn0;
        m1 = mn1;
        float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float p = expf(__fsub_rn(sacc[4 * j + i], (i >> 1) ? mn1 : mn0));
                sacc[4 * j + i] = p;
                if (i >> 1) rs1 = __fadd_rn(rs1, p);
                else rs0 = __fadd_rn(rs0, p);
            }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
            rs0 = __fadd_rn(rs0, __shfl_xor_sync(0xffffffffu, rs0, off));
            rs1 = __fadd_rn(rs1, __shfl_xor_sync(0xffffffffu, rs1, off));
        }
        l0 = __fadd_rn(__fmul_rn(l0, al0), rs0);
        l1 = __fadd_rn(__fmul_rn(l1, al1), rs1);
#pragma unroll
        for (int i = 0; i < D / 2; ++i) oacc[i] = __fmul_rn(oacc[i], (i & 2) ? al1 : al0);

        // P's A fragments from the accumulator layout: k-step kk covers keys 16 kk .. 16 kk + 15 of the tile
        uint32_t pa1[4][4], pa2[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int f = 0; f < 4; ++f) split_bf16x2(sacc[8 * kk + 2 * f], sacc[8 * kk + 2 * f + 1], pa1[kk][f], pa2[kk][f]);

        // O += P V
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint64_t d1 = make_smem_desc_none(v_hi_a + 256 * kk, 128, 1024);
            const uint64_t d2 = make_smem_desc_none(v_lo_a + 256 * kk, 128, 1024);
            Wgmma<D, 0>::mma(oacc, pa2[kk], d1, 1u);  // p2 * v1
            Wgmma<D, 0>::mma(oacc, pa1[kk], d2, 1u);  // p1 * v2
            Wgmma<D, 0>::mma(oacc, pa1[kk], d1, 1u);  // p1 * v1
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
    }

    // O / l; oacc[4j + i] is row (i >> 1 ? r1 : r0), column 8j + 2c + (i & 1)
    const int e = heads * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int row = (i >> 1) ? r1 : r0;
            if (row < lq)
                o[(static_cast<size_t>(b) * lq + row) * e + h * D + 8 * j + 2 * c + (i & 1)] =
                    __fdiv_rn(oacc[4 * j + i], (i >> 1) ? l1 : l0);
        }
}

template <int D>
static int attention_launch(float* o, const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                            int batch, int heads, int lq, int lk, float scale, cudaStream_t s) {
    static SmemAttrCache cache;
    constexpr int smem = attn_smem_bytes<D>();
    if (int rc = ensure_dynamic_smem(attention_kernel<D>, smem, cache)) return rc;
    const dim3 grid(static_cast<unsigned>(batch), static_cast<unsigned>(heads * ((lq + kAttnBM - 1) / kAttnBM)));
    attention_kernel<D><<<grid, kAttnThreads, smem, s>>>(o, q, ldq, k, ldk, v, ldv, heads, lq, lk, scale);
    return 0;
}

int attention(float* o, const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, int batch,
              int heads, int d, int lq, int lk, float scale, cudaStream_t s) {
    const double n = static_cast<double>(batch) * heads;
    const double flops = 4.0 * n * lq * static_cast<double>(lk) * d;
    const double bytes = 4.0 * n * d * (2.0 * lq + 2.0 * lk);
    const int prof = prof_begin(s, PROF_ATTENTION, flops, 3.0 * flops, bytes);
    int rc;
    switch (d) {
        case 16: rc = attention_launch<16>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
        case 32: rc = attention_launch<32>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
        case 48: rc = attention_launch<48>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
        case 64: rc = attention_launch<64>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
        case 80: rc = attention_launch<80>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
        case 96: rc = attention_launch<96>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
        case 112: rc = attention_launch<112>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
        default: rc = attention_launch<128>(o, q, ldq, k, ldk, v, ldv, batch, heads, lq, lk, scale, s); break;
    }
    prof_end(prof, s);
    if (rc) return rc;
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
