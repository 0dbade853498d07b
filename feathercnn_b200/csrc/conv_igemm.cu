// SGECONV — implicit-GEMM convolution straight from the NCHW blob on Hopper warpgroup MMA (sm_90a).
//
// Replaces the idea of the reference's SGECONV algorithm ("packs B directly from the padded input, no materialised
// im2col"; a stub in its AVX dispatcher) and of im2col + packed SGEMM with a formulation that has NO intermediate in HBM
// and no A tile in shared memory:
//
//   D[pixel][oc] = sum_k  A[pixel][k] * Wp[oc][k],    k = (u*KW + v)*IC + ic   (IC % 32 != 0)
//                                                      k = ((ic/32)*KH*KW + u*KW + v)*32 + ic%32   (IC % 32 == 0: a k-block
//                                                      is one tap x 32 channels -> one bounds check per pixel and k-block)
//   A[pixel][k]  = X[n][ic][oy*s+u*d-pad][ox*s+v*d-pad]   (0 outside the image: the im2col rule)
//
//   M tile     = 128 output pixels, consecutive along the flattened (n, oy, ox) index; with a fused 2x2 max pooling a
//                2-row x 64-column patch instead, laid out so that the four pixels of a pooling window sit in one thread
//                (rows g, g + 8 of its fragment) and its neighbour lane (lane ^ 4).
//   A operand  = gathered by the consumer threads straight from global memory into the registers of their wgmma
//                fragment (the next k-block's loads are in flight while the current one is multiplied), split on chip:
//                PLANES 3 (default) BF16x3 — x = p1 + p2 + r with p1 = RN_bf16(x), p2 = RN_bf16(x - p1), three bf16 MMAs
//                p2*q1 + p1*q2 + p1*q1 per k-step of 16; 2 = 3xTF32 (hi = x & 0xFFFFE000, lo = x - hi, three tf32 MMAs per
//                k-step of 8); 1 = plain TF32.
//   B operand  = filters re-packed once at Init, K-major.  BF16x3: two bf16 planes PRE-TILED in global memory in the
//                un-swizzled core-matrix order of wgmma, [k-block][N tile][plane][row/8][16-byte k chunk][row%8][8]: a ring
//                stage is one contiguous run fetched by ONE cp.async.bulk.  3xTF32 / TF32: Wp[oc][k] fp32 rows (hi / lo
//                planes), TMA tensor loads with the 128-byte swizzle.  A producer warp keeps a 4-deep ring ahead.
//   MMA        = wgmma.mma_async, A from registers, B from shared memory, fp32 register accumulators (two warpgroups of
//                64 pixels).
//   epilogue   = +bias [+ residual: fused Eltwise SUM] -> ReLU [-> 2x2 max pooling by one shuffle] -> NCHW stores.
//
// Used where non-fused Winograd is bandwidth-bound (large images, <= 128 channels) and for every layer the reference
// sends to im2col + SGEMM (1x1, strided, 7x7, IC = 3, small images).
#include "conv_igemm.cuh"

#include "common.cuh"

#include <stdlib.h>
#include <string.h>
#include "wgmma.cuh"
#include <cuda_bf16.h>

namespace fcuda {

namespace {

constexpr int kConsumerWarps = 8;                      // two warpgroups x 64 pixels
constexpr int kThreadsIg = (kConsumerWarps + 1) * 32;  // + the filter producer warp
constexpr int kStagesIg = 4;
constexpr int kMaxTableK = 6144;                       // k-table entries that fit beside the filter ring

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

struct IgemmArgs {
    const float* residual;   // added to the output before the activation, or null
    const float* in;
    float* out;
    const float* bias;
    int N, IC, H, W, OC, OH, OW;
    int KH, KW, pad_top, pad_left, stride_h, stride_w;
    int dil_h, dil_w;        // tap spacing (1 = dense)
    int in_img_c, out_img_c; // channels per image of the tensors `in` / `out` point into (>= IC / OC: channel slices)
    int K;                   // KH*KW*IC
    int kblocks;             // ceil(K / 32)
    int use_table;           // 0 => IC % 32 == 0: every k-block is 32 channels of ONE tap, offsets are arithmetic
    int taps;                // KH*KW
    int num_n;               // ceil(OC / BN)
    long long total_pix;     // N * OH * OW
    int relu;
    int pool;                // fuse a following 2x2 / stride-2 max pooling; `out` is the pooled blob
    int tiles_x, tiles_y;    // pool: 64-column x 2-row patches per image
    const unsigned char* wbf;  // BF16x3: pre-tiled filter planes (see igemm_pack_weights_bf16_kernel)
    unsigned wbf_kb_bytes;     // bytes of one k-block (both planes, every N tile): 2 * ocpad * 64
};

// The k index (inside a 32-wide k-block) of fragment element j of lane column c: tf32 k-steps of 8 hold (c, c + 4),
// bf16 k-steps of 16 hold the pairs (2c, 2c + 1) and (2c + 8, 2c + 9).
template <bool BF>
__device__ __forceinline__ int frag_k(int j, int c) {
    return BF ? (j >> 2) * 16 + 2 * c + (j & 1) + 8 * ((j >> 1) & 1) : (j >> 1) * 8 + c + 4 * (j & 1);
}

template <int BN, int PLANES>
__global__ void __launch_bounds__(kThreadsIg, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmWlo,
                  const IgemmArgs args) {
    constexpr bool BF = PLANES == 3;
    constexpr int NPL = BF ? 2 : PLANES;                  // operand planes in memory
    constexpr int kBTile = BN * 32 * (BF ? 2 : 4);        // 32 k-values per row: 128 B of fp32 / 64 B of bf16
    constexpr int kStage = NPL * kBTile;                  // [B_hi][B_lo]
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    int2* ktab = reinterpret_cast<int2*>(smem + kStagesIg * kStage);  // use_table: {element offset, dy << 16 | dx} per k
    __shared__ uint64_t full_bar[kStagesIg];
    __shared__ uint64_t empty_bar[kStagesIg];

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_blk = static_cast<int>(blockIdx.x % static_cast<unsigned>(args.num_n));
    const long long ptile = blockIdx.x / static_cast<unsigned>(args.num_n);
    const int kblocks = args.kblocks;
    const int plane = args.H * args.W;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStagesIg; ++s) {
            ptx::mbar_init(&full_bar[s], 1);
            ptx::mbar_init(&empty_bar[s], kConsumerWarps);
        }
        ptx::fence_barrier_init();
    }
    if (args.use_table) {
        for (int k = threadIdx.x; k < kblocks * 32; k += kThreadsIg) {
            int2 e = make_int2(0, 0);
            if (k < args.K) {
                const int tap = k / args.IC, ic = k - tap * args.IC;
                const int dy = (tap / args.KW) * args.dil_h, dx = (tap % args.KW) * args.dil_w;
                e = make_int2(ic * plane + dy * args.W + dx, (dy << 16) | dx);
            }
            ktab[k] = e;
        }
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ===================== filter producer =====================
        if (lane == 0) {
            if (!BF) {
                ptx::prefetch_tensormap(&tmW);
                if (NPL == 2) ptx::prefetch_tensormap(&tmWlo);
            }
            for (int kb = 0; kb < kblocks; ++kb) {
                const int stage = kb % kStagesIg;
                if (kb >= kStagesIg) ptx::mbar_wait_nocall(&empty_bar[stage], ((kb / kStagesIg) - 1) & 1);
                uint8_t* st = smem + stage * kStage;
                ptx::mbar_arrive_expect_tx(&full_bar[stage], kStage);
                if (BF) {
                    ptx::bulk_load_1d(st, args.wbf + static_cast<size_t>(kb) * args.wbf_kb_bytes + static_cast<size_t>(n_blk) * kStage,
                                      kStage, &full_bar[stage]);
                } else {
                    ptx::tma_load_3d(st, &tmW, &full_bar[stage], kb * 32, n_blk * BN, 0);
                    if (NPL == 2) ptx::tma_load_3d(st + kBTile, &tmWlo, &full_bar[stage], kb * 32, n_blk * BN, 0);
                }
            }
        }
        return;
    }

    // ===================== consumers =====================
    const int gq = lane >> 2, c = lane & 3;
    // the two pixels (fragment rows gq, gq + 8 of this warp's 16) this thread gathers and stores
    int img[2], oy[2], ox[2];
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (args.pool) {
            const int per_img = args.tiles_x * args.tiles_y;
            const int n = static_cast<int>(ptile / per_img);
            const int rem = static_cast<int>(ptile - static_cast<long long>(n) * per_img);
            const int ty = rem / args.tiles_x, tx = rem - ty * args.tiles_x;
            img[h] = n;
            oy[h] = 2 * ty + h;
            ox[h] = 64 * tx + 8 * warp + gq;
            valid[h] = oy[h] < args.OH && ox[h] < args.OW;
        } else {
            const long long m = ptile * 128 + warp * 16 + 8 * h + gq;
            valid[h] = m < args.total_pix;
            const long long mm = valid[h] ? m : 0;
            const int pix_per_img = args.OH * args.OW;
            img[h] = static_cast<int>(mm / pix_per_img);
            const int pix = static_cast<int>(mm - static_cast<long long>(img[h]) * pix_per_img);
            oy[h] = pix / args.OW;
            ox[h] = pix - oy[h] * args.OW;
        }
    }
    int iy0[2], ix0[2];
    long long ibase[2];  // element offset of tap (0, 0), channel 0 of the pixel's receptive field
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        iy0[h] = oy[h] * args.stride_h - args.pad_top;
        ix0[h] = ox[h] * args.stride_w - args.pad_left;
        ibase[h] = static_cast<long long>(img[h]) * args.in_img_c * plane + static_cast<long long>(iy0[h]) * args.W + ix0[h];
    }
    const float* __restrict__ in = args.in;

    // raw A values of one k-block: [row h][fragment element j]
    auto gather = [&](int kb, float (&raw)[2][8]) {
        if (!args.use_table) {
            const int cb = kb / args.taps, tap = kb - cb * args.taps;
            const int dy = (tap / args.KW) * args.dil_h, dx = (tap % args.KW) * args.dil_w;
            const long long koff = static_cast<long long>(cb) * 32 * plane + dy * args.W + dx;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const bool ok = valid[h] && static_cast<unsigned>(iy0[h] + dy) < static_cast<unsigned>(args.H) &&
                                static_cast<unsigned>(ix0[h] + dx) < static_cast<unsigned>(args.W);
                const float* p = in + (ok ? ibase[h] + koff : 0);
#pragma unroll
                for (int j = 0; j < 8; ++j) raw[h][j] = ok ? __ldg(p + static_cast<size_t>(frag_k<BF>(j, c)) * plane) : 0.f;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int k = kb * 32 + frag_k<BF>(j, c);
                int2 e;
                asm volatile("ld.shared.v2.s32 {%0, %1}, [%2];" : "=r"(e.x), "=r"(e.y) : "r"(ptx::smem_u32(ktab + k)));
                const int dy = e.y >> 16, dx = e.y & 0xFFFF;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const bool ok = valid[h] && k < args.K && static_cast<unsigned>(iy0[h] + dy) < static_cast<unsigned>(args.H) &&
                                    static_cast<unsigned>(ix0[h] + dx) < static_cast<unsigned>(args.W);
                    raw[h][j] = ok ? __ldg(in + ibase[h] + e.x) : 0.f;
                }
            }
        }
    };

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    float raw[2][8];
    gather(0, raw);
    for (int kb = 0; kb < kblocks; ++kb) {
        const int stage = kb % kStagesIg;
        // split this k-block's operand into the fragments, then start the next k-block's loads
        uint32_t f1[4][4], f2[4][4];  // [k-step][a0..a3]: hi / p1 and lo / p2
        if (BF) {
#pragma unroll
            for (int kk = 0; kk < 2; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q) {  // a0 (row gq, pair 0), a1 (row gq + 8, pair 0), a2 (gq, pair 1), a3 (gq + 8, pair 1)
                    const int h = q & 1, j = 4 * kk + 2 * (q >> 1);
                    split_bf16x2(raw[h][j], raw[h][j + 1], f1[kk][q], f2[kk][q]);
                }
        } else {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float x = raw[q & 1][2 * kk + (q >> 1)];
                    if (PLANES == 2) split_tf32_trunc(x, f1[kk][q], f2[kk][q]);
                    else f1[kk][q] = __float_as_uint(x);
                }
        }
        if (kb + 1 < kblocks) gather(kb + 1, raw);
        ptx::mbar_wait_nocall(&full_bar[stage], (kb / kStagesIg) & 1);
        const uint32_t b_base = ptx::smem_u32(smem + stage * kStage);
        ptx::wgmma_fence();
        if (BF) {
            // un-swizzled core matrices: LBO = 128 B between k chunks, SBO = 512 B between 8-row groups; a k-step = 2 chunks
            const uint64_t dQ1 = make_smem_desc_none(b_base, 128, 512);
            const uint64_t dQ2 = make_smem_desc_none(b_base + kBTile, 128, 512);
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                Wgmma<BN, 0>::mma(acc, f2[kk], dQ1 + 16 * kk, 1u);  // p2 * q1
                Wgmma<BN, 0>::mma(acc, f1[kk], dQ2 + 16 * kk, 1u);  // p1 * q2
                Wgmma<BN, 0>::mma(acc, f1[kk], dQ1 + 16 * kk, 1u);  // p1 * q1
            }
        } else {
            const uint64_t dB = make_smem_desc_sw128(b_base);
            const uint64_t dBlo = make_smem_desc_sw128(b_base + kBTile);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                if (PLANES == 2) {
                    Wgmma<BN, 1>::mma(acc, f2[kk], dB + 2 * kk, 1u);    // A_lo * B_hi
                    Wgmma<BN, 1>::mma(acc, f1[kk], dBlo + 2 * kk, 1u);  // A_hi * B_lo
                    Wgmma<BN, 1>::mma(acc, f1[kk], dB + 2 * kk, 1u);    // A_hi * B_hi
                } else {
                    Wgmma<BN, 1>::mma(acc, f1[kk], dB + 2 * kk, 1u);
                }
            }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty_bar[stage]);
    }

    // ===================== epilogue =====================
    const int oplane = args.OH * args.OW;
    const int SH = (args.OH + 1) >> 1, SW = (args.OW + 1) >> 1;  // pooled geometry
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int oc = n_blk * BN + 8 * j + 2 * c + e;
            const bool oc_ok = oc < args.OC;
            const float bv = (args.bias != nullptr && oc_ok) ? __ldg(args.bias + oc) : 0.f;
            float v[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                v[h] = acc[4 * j + 2 * h + e] + bv;
                const size_t o = (static_cast<size_t>(img[h]) * args.out_img_c + oc) * oplane + static_cast<size_t>(oy[h]) * args.OW + ox[h];
                if (args.residual != nullptr && valid[h] && oc_ok) v[h] += __ldg(args.residual + o);
                if (args.relu) v[h] = fmaxf(v[h], 0.f);
                if (!args.pool && valid[h] && oc_ok) args.out[o] = v[h];
            }
            if (args.pool) {
                float m = fmaxf(valid[0] ? v[0] : -INFINITY, valid[1] ? v[1] : -INFINITY);
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));  // the window's other column: pixel gq ^ 1
                if ((gq & 1) == 0 && valid[0] && oc_ok)
                    args.out[(static_cast<size_t>(img[0]) * args.out_img_c + oc) * (static_cast<size_t>(SH) * SW) +
                             static_cast<size_t>(oy[0] >> 1) * SW + (ox[0] >> 1)] = m;
            }
        }
    }
}

// W[oc][ic][tap] -> Wp[oc][Kf] hi/lo planes, k = tap*IC + ic, Kf = K rounded up to 4 (TMA's 16-byte row rule)
__global__ void __launch_bounds__(256)
igemm_pack_weights_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int OC, int IC,
                          int taps, int Kf) {
    const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const size_t total = static_cast<size_t>(OC) * Kf;
    if (idx >= total) return;
    const int k = static_cast<int>(idx % Kf);
    const int oc = static_cast<int>(idx / Kf);
    float v = 0.f;
    if (k < IC * taps) {
        int tap, ic;
        if (IC % 32 == 0) {  // k = (cb * taps + tap) * 32 + ic % 32
            const int kb = k >> 5;
            const int cb = kb / taps;
            tap = kb - cb * taps;
            ic = cb * 32 + (k & 31);
        } else {             // k = tap * IC + ic
            tap = k / IC;
            ic = k - tap * IC;
        }
        v = w[(static_cast<size_t>(oc) * IC + ic) * taps + tap];
    }
    if (lo) {
        float h, l;
        split_tf32(v, h, l);
        hi[idx] = h;
        lo[idx] = l;
    } else {
        hi[idx] = v;
    }
}

// BF16x3: two bf16 planes q1 = RN(w), q2 = RN(w - q1), PRE-TILED for the kernel's filter ring, ordered
//     [k-block kb (32 k-values, same k order as above)][N tile nb (BN rows)][plane][row / 8][16-byte k chunk (4)][row % 8][8 bf16]
// i.e. per (k-block, N tile) both planes are ONE contiguous run of 8-row x 16-byte core matrices — the un-swizzled K-major
// shared-memory layout of wgmma — so the kernel fetches a ring stage with one 1-D bulk copy.  Rows >= OC and k >= K are
// zeros; BN = the N tile the dispatcher picks for this OC, OCpad = OC rounded up to it.
__global__ void __launch_bounds__(256)
igemm_pack_weights_bf16_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ q, int OC, int IC, int taps, int KB,
                               int OCpad, int BN) {
    const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;  // over [kb][oc][kk]
    const size_t total = static_cast<size_t>(KB) * OCpad * 32;
    if (idx >= total) return;
    const int kk = static_cast<int>(idx & 31);
    const int oc = static_cast<int>((idx >> 5) % OCpad);
    const int kb = static_cast<int>((idx >> 5) / OCpad);
    const int k = kb * 32 + kk;
    float v = 0.f;
    if (oc < OC && k < IC * taps) {
        int tap, ic;
        if (IC % 32 == 0) {
            const int cb = kb / taps;
            tap = kb - cb * taps;
            ic = cb * 32 + kk;
        } else {
            tap = k / IC;
            ic = k - tap * IC;
        }
        v = w[(static_cast<size_t>(oc) * IC + ic) * taps + tap];
    }
    const __nv_bfloat16 a = __float2bfloat16_rn(v);
    const int nb = oc / BN, r = oc - nb * BN;
    const size_t tile = (static_cast<size_t>(kb) * (OCpad / BN) + nb) * 2 * BN * 32;  // elements before this (k-block, N tile)
    const size_t dst = tile + static_cast<size_t>(r & ~7) * 32 + (kk >> 3) * 64 + (r & 7) * 8 + (kk & 7);
    q[dst] = a;
    q[dst + static_cast<size_t>(BN) * 32] = __float2bfloat16_rn(v - __bfloat162float(a));
}


// N tile conv_igemm_forward uses for a layer with OC output channels and the padded row count of the tiled planes
static int igemm_bn_for(int OC) { return OC <= 32 ? 32 : OC <= 64 ? 64 : 128; }
static int igemm_ocpad(int OC) { const int bn = igemm_bn_for(OC); return (OC + bn - 1) / bn * bn; }

template <int BN, int PLANES>
int launch_igemm(const IgemmProblem& p, cudaStream_t stream) {
    constexpr bool BF = PLANES == 3;
    constexpr int NPL = BF ? 2 : PLANES;
    const int taps = p.KH * p.KW;
    const int K = taps * p.IC;
    CUtensorMap tmW, tmWlo;
    memset(&tmW, 0, sizeof(tmW));
    tmWlo = tmW;
    if (!BF) {  // the BF16x3 planes are pre-tiled and fetched by 1-D bulk copies: no tensor map
        EncodeTiledFn enc = encode_fn();
        if (!enc) return FCUDA_ERR_CUDA;
        const int Kf = (K + 3) & ~3;
        for (int pl = 0; pl < NPL; ++pl) {
            cuuint64_t dims[3] = {(cuuint64_t)Kf, (cuuint64_t)p.OC, 1};
            cuuint64_t strides[2] = {(cuuint64_t)Kf * 4, (cuuint64_t)Kf * p.OC * 4};
            cuuint32_t box[3] = {32, (cuuint32_t)BN, 1};
            cuuint32_t estr[3] = {1, 1, 1};
            const float* base = pl == 0 ? p.w_hi : p.w_lo;
            CUresult r = enc(pl == 0 ? &tmW : &tmWlo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides,
                             box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
                fprintf(stderr, "fcuda: igemm weight tensor map failed (%d)\n", (int)r);
                return FCUDA_ERR_CUDA;
            }
        }
    }
    IgemmArgs a;
    a.wbf = reinterpret_cast<const unsigned char*>(p.w_hi);
    a.wbf_kb_bytes = 2u * static_cast<unsigned>(igemm_ocpad(p.OC)) * 64u;
    if (BF && (igemm_bn_for(p.OC) != BN || static_cast<unsigned long long>(ceil_div(K, 32)) * igemm_ocpad(p.OC) * 128ull >= (1ull << 31))) return -1;
    a.in = p.input; a.out = p.output; a.bias = p.bias; a.residual = p.residual;
    a.N = p.N; a.IC = p.IC; a.H = p.H; a.W = p.W; a.OC = p.OC; a.OH = p.OH; a.OW = p.OW;
    a.KH = p.KH; a.KW = p.KW; a.pad_top = p.pad_top; a.pad_left = p.pad_left;
    a.stride_h = p.stride_h; a.stride_w = p.stride_w;
    a.dil_h = p.dil_h > 1 ? p.dil_h : 1; a.dil_w = p.dil_w > 1 ? p.dil_w : 1;
    a.in_img_c = p.in_c_total > 0 ? p.in_c_total : p.IC;
    a.out_img_c = p.out_c_total > 0 ? p.out_c_total : p.OC;
    a.K = K;
    a.kblocks = ceil_div(K, 32);
    a.use_table = (p.IC % 32 == 0) ? 0 : 1;
    a.taps = taps;
    a.num_n = ceil_div(p.OC, BN);
    a.total_pix = static_cast<long long>(p.N) * p.OH * p.OW;
    a.relu = p.relu;
    a.pool = p.pool ? 1 : 0;
    a.tiles_x = ceil_div(p.OW, 64);
    a.tiles_y = ceil_div(p.OH, 2);
    const long long pixel_tiles = a.pool ? static_cast<long long>(p.N) * a.tiles_x * a.tiles_y : (a.total_pix + 127) / 128;
    const long long total = pixel_tiles * a.num_n;
    // 32-bit plane strides and packed tap offsets (dy << 16 | dx) inside the kernel; the k-table's element offsets
    // ic * H * W + dy * W + dx are 32-bit as well
    const long long table_max = static_cast<long long>(p.IC - 1) * p.H * p.W + static_cast<long long>(p.KH - 1) * a.dil_h * p.W +
                                static_cast<long long>(p.KW - 1) * a.dil_w;
    if (total >= (1ll << 31) || static_cast<long long>(p.H) * p.W >= (1ll << 30) || static_cast<long long>(p.OH) * p.OW >= (1ll << 30) ||
        (p.KH - 1) * a.dil_h >= (1 << 15) || (p.KW - 1) * a.dil_w >= (1 << 16) || (a.use_table && table_max >= (1ll << 31)))
        return -1;
    constexpr int kStage = NPL * BN * 32 * (BF ? 2 : 4);
    const int table_bytes = a.use_table ? a.kblocks * 32 * 8 : 0;
    const int smem = kStagesIg * kStage + table_bytes + 1024;
    if (smem > 227 * 1024) return -1;
    auto kern = conv_igemm_kernel<BN, PLANES>;
    static SmemAttrCache attr_cache;
    if (int rc = ensure_dynamic_smem(kern, smem, attr_cache)) return rc;
    // algorithmic work of the layer: direct-convolution FLOPs; input + filters read once, output written once
    const double macs = static_cast<double>(p.N) * p.OC * p.OH * p.OW * p.IC * taps;
    const double mma = 2.0 * static_cast<double>(pixel_tiles) * 128 * (a.num_n * BN) * (a.kblocks * 32) * (PLANES >= 2 ? 3 : 1);
    const int prof = prof_begin(stream, PROF_IGEMM, 2.0 * macs, mma,
                                4.0 * (static_cast<double>(p.N) * p.IC * p.H * p.W + static_cast<double>(p.OC) * K +
                                       static_cast<double>(p.N) * p.OC * p.OH * p.OW * (p.residual ? 2 : 1)));
    kern<<<static_cast<unsigned>(total), kThreadsIg, smem, stream>>>(tmW, tmWlo, a);
    prof_end(prof, stream);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

// ===================================================================================================================
// Halo kernel: stride-1, dense layers with IC % 32 == 0 (k = ((ic/32)*taps + tap)*32 + ic%32, as above).
//
//   M tile     = an R x C patch of output pixels inside one image (R * C = 128, C in {8, 16, 32, 64}); warp w covers rows
//                2*(w / (C/8)) + {0, 1} (fragment rows gq, gq + 8) and columns 8*(w % (C/8)) + gq, so a fused 2x2 pooling
//                window still sits in one thread and its lane ^ 4 neighbour.
//   A operand  = per 32-channel block ONE 4-D TMA box {Cb, Rb, 32, 1} of the input blob at (x0 - xpad, y0 - pad_top),
//                xpad = pad_left rounded up to 4 so that every box row starts on a 16-byte boundary: the patch plus its
//                halo, zero-filled outside the image (= the im2col padding).  Every tap (dy, dx) of the
//                block reads it as a shifted view with ld.shared, so each input value crosses L2 -> SM once per channel
//                block instead of once per tap.  Boxes have their own 2-deep ring; Rb / Cb are padded until the warp's 32
//                words of one gather (8 columns x 4 channel planes) hit 32 different banks (halo_banks_conflict_free).
//   B operand  = the same pre-tiled filter planes / swizzled TMA rows and the same 4-deep ring as conv_igemm_kernel.
//   pipeline   = two fragment sets: k-block kb + 1 is gathered and split while kb's wgmma group runs (wgmma_wait<1>); a
//                filter stage is released once its group retired.  Persistent CTAs loop over tiles, so the producer warp
//                fetches the next tile's halo and filters during the epilogue.
//
// Per k-block the wgmma sequence (p2*q1, p1*q2, p1*q1 per k-step), the operand values, the k order and BN are those of
// conv_igemm_kernel: the result is bit-identical to it.
constexpr int kHaloStages = 2;

struct HaloArgs {
    const float* residual;
    float* out;
    const float* bias;
    int OC, OH, OW, KW, taps;
    int out_img_c;
    int kblocks, num_n;
    int relu, pool;
    int R, C;              // output patch rows x columns (128 pixels)
    int tiles_x, tiles_y;  // patches per image
    int Rb, Cb;            // halo box rows / columns in shared memory (padded)
    int pad_top, xpad;     // box origin relative to the patch: rows -pad_top, columns -xpad (xpad % 4 == 0)
    int xshift;            // xpad - pad_left: box column of tap dx = 0 for patch column 0
    long long tiles;       // N * tiles_y * tiles_x * num_n
    const unsigned char* wbf;
    unsigned wbf_kb_bytes;
    int pr, pc;            // conv_igemm_presplit_kernel: rows x columns of the bf16 planes (R + KH - 1, C + KW - 1)
};

// Epilogue of the halo kernels for one m64 accumulator (as conv_igemm_kernel): this thread's pixels are rows oy[0..1]
// of column ox in image img.
template <int BN>
__device__ __forceinline__ void halo_epilogue(const float (&acc)[BN / 2], const HaloArgs& args, int n_blk, int img,
                                              const int (&oy)[2], const bool (&valid)[2], int ox, int oplane, int SH,
                                              int SW, int c, int gq) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int oc = n_blk * BN + 8 * j + 2 * c + e;
            const bool oc_ok = oc < args.OC;
            const float bv = (args.bias != nullptr && oc_ok) ? __ldg(args.bias + oc) : 0.f;
            float v[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                v[h] = acc[4 * j + 2 * h + e] + bv;
                const size_t o = (static_cast<size_t>(img) * args.out_img_c + oc) * oplane + static_cast<size_t>(oy[h]) * args.OW + ox;
                if (args.residual != nullptr && valid[h] && oc_ok) v[h] += __ldg(args.residual + o);
                if (args.relu) v[h] = fmaxf(v[h], 0.f);
                if (!args.pool && valid[h] && oc_ok) args.out[o] = v[h];
            }
            if (args.pool) {
                float m = fmaxf(valid[0] ? v[0] : -INFINITY, valid[1] ? v[1] : -INFINITY);
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));  // the window's other column: pixel gq ^ 1
                if ((gq & 1) == 0 && valid[0] && oc_ok)
                    args.out[(static_cast<size_t>(img) * args.out_img_c + oc) * (static_cast<size_t>(SH) * SW) +
                             static_cast<size_t>(oy[0] >> 1) * SW + (ox >> 1)] = m;
            }
        }
    }
}

// Producer warp of the halo kernels (lane 0 only): the HS-deep ring of input boxes and the filter ring, in consumption
// order.  A tile is args.R x args.C output pixels; its box for channel block cb starts at (x0 - xpad, y0 - pad_top).
template <int BN, int PLANES, int HS>
__device__ __forceinline__ void halo_producer(const CUtensorMap* tmX, const CUtensorMap* tmW, const CUtensorMap* tmWlo,
                                              const HaloArgs& args, uint8_t* smem, float* halo, int hstage,
                                              uint64_t* full_bar, uint64_t* empty_bar, uint64_t* hfull_bar,
                                              uint64_t* hempty_bar) {
    constexpr bool BF = PLANES == 3;
    constexpr int NPL = BF ? 2 : PLANES;
    constexpr int kBTile = BN * 32 * (BF ? 2 : 4);
    constexpr int kStage = NPL * kBTile;
    const int per_img = args.tiles_x * args.tiles_y;
    const int taps = args.taps;
    const int ncb = args.kblocks / taps;
    ptx::prefetch_tensormap(tmX);
    if (!BF) {
        ptx::prefetch_tensormap(tmW);
        if (NPL == 2) ptx::prefetch_tensormap(tmWlo);
    }
    int hb = 0;   // boxes issued
    int kbg = 0;  // filter stages issued
    auto load_halo = [&](long long t, int cb) {
        const long long pt = t / args.num_n;
        const int n = static_cast<int>(pt / per_img);
        const int rem = static_cast<int>(pt - static_cast<long long>(n) * per_img);
        const int ty = rem / args.tiles_x, tx = rem - ty * args.tiles_x;
        const int hs = hb % HS;
        if (hb >= HS) ptx::mbar_wait_nocall(&hempty_bar[hs], ((hb / HS) - 1) & 1);
        ptx::mbar_arrive_expect_tx(&hfull_bar[hs], static_cast<uint32_t>(hstage) * 4u);
        ptx::tma_load_4d(halo + hs * hstage, tmX, &hfull_bar[hs], tx * args.C - args.xpad, ty * args.R - args.pad_top,
                         cb * 32, n);
        ++hb;
    };
    if (blockIdx.x < args.tiles) load_halo(blockIdx.x, 0);
    for (long long t = blockIdx.x; t < args.tiles; t += gridDim.x) {
        const int n_blk = static_cast<int>(t % args.num_n);
        for (int cb = 0, kb = 0; cb < ncb; ++cb) {
            for (int tap = 0; tap < taps; ++tap, ++kb, ++kbg) {
                const int stage = kbg % kStagesIg;
                if (kbg >= kStagesIg) ptx::mbar_wait_nocall(&empty_bar[stage], ((kbg / kStagesIg) - 1) & 1);
                uint8_t* st = smem + stage * kStage;
                ptx::mbar_arrive_expect_tx(&full_bar[stage], kStage);
                if (BF) {
                    ptx::bulk_load_1d(st, args.wbf + static_cast<size_t>(kb) * args.wbf_kb_bytes + static_cast<size_t>(n_blk) * kStage,
                                      kStage, &full_bar[stage]);
                } else {
                    ptx::tma_load_3d(st, tmW, &full_bar[stage], kb * 32, n_blk * BN, 0);
                    if (NPL == 2) ptx::tma_load_3d(st + kBTile, tmWlo, &full_bar[stage], kb * 32, n_blk * BN, 0);
                }
                if (tap == 0) {  // the next box (this tile's next channel block or the next tile's first) lands meanwhile
                    if (cb + 1 < ncb) load_halo(t, cb + 1);
                    else if (t + gridDim.x < args.tiles) load_halo(t + gridDim.x, 0);
                }
            }
        }
    }
}

template <int BN, int PLANES>
__global__ void __launch_bounds__(kThreadsIg, 1)
conv_igemm_halo_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                       const __grid_constant__ CUtensorMap tmWlo, const HaloArgs args) {
    constexpr bool BF = PLANES == 3;
    constexpr int NPL = BF ? 2 : PLANES;
    constexpr int kBTile = BN * 32 * (BF ? 2 : 4);
    constexpr int kStage = NPL * kBTile;
    extern __shared__ uint8_t smem_raw[];
    // indexing smem_raw itself (not a re-cast integer) keeps the halo reads ld.shared
    uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
    const float* halo = reinterpret_cast<const float*>(smem + kStagesIg * kStage);
    const int cstride = args.Rb * args.Cb;  // floats between the channel planes of a box
    const int hstage = 32 * cstride;        // floats per box
    __shared__ uint64_t full_bar[kStagesIg];
    __shared__ uint64_t empty_bar[kStagesIg];
    __shared__ uint64_t hfull_bar[kHaloStages];
    __shared__ uint64_t hempty_bar[kHaloStages];

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int per_img = args.tiles_x * args.tiles_y;
    const int kblocks = args.kblocks, taps = args.taps;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStagesIg; ++s) {
            ptx::mbar_init(&full_bar[s], 1);
            ptx::mbar_init(&empty_bar[s], kConsumerWarps);
        }
        for (int s = 0; s < kHaloStages; ++s) {
            ptx::mbar_init(&hfull_bar[s], 1);
            ptx::mbar_init(&hempty_bar[s], kConsumerWarps);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ===================== producer: halo boxes + filters, in consumption order =====================
        if (lane == 0)
            halo_producer<BN, PLANES, kHaloStages>(&tmX, &tmW, &tmWlo, args, smem, const_cast<float*>(halo), hstage, full_bar,
                                                   empty_bar, hfull_bar, hempty_bar);
        return;
    }

    // ===================== consumers =====================
    const int gq = lane >> 2, c = lane & 3;
    const int wcols = args.C >> 3;
    const int wy = warp / wcols, wx = warp - wy * wcols;
    const int prow = 2 * wy, pcol = 8 * wx + gq;  // this thread's pixels in the patch: rows prow + h, column pcol
    // word offset of (channel frag_k(0, c), row prow, column pcol) inside a box; tap (dy, dx) adds dy * Cb + dx
    const int abase = (BF ? 2 * c : c) * cstride + prow * args.Cb + pcol + args.xshift;

    auto gather = [&](const float* box, int toff, float (&raw)[2][8]) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 8; ++j) raw[h][j] = box[abase + toff + h * args.Cb + frag_k<BF>(j, 0) * cstride];
    };
    auto split = [&](const float (&raw)[2][8], uint32_t (&f1)[4][4], uint32_t (&f2)[4][4]) {
        if (BF) {
#pragma unroll
            for (int kk = 0; kk < 2; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int h = q & 1, j = 4 * kk + 2 * (q >> 1);
                    split_bf16x2(raw[h][j], raw[h][j + 1], f1[kk][q], f2[kk][q]);
                }
        } else {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float x = raw[q & 1][2 * kk + (q >> 1)];
                    if (PLANES == 2) split_tf32_trunc(x, f1[kk][q], f2[kk][q]);
                    else f1[kk][q] = __float_as_uint(x);
                }
        }
    };

    const int oplane = args.OH * args.OW;
    const int SH = (args.OH + 1) >> 1, SW = (args.OW + 1) >> 1;  // pooled geometry
    int kbg = 0;  // filter stages consumed
    int hb = 0;   // boxes consumed
    for (long long t = blockIdx.x; t < args.tiles; t += gridDim.x) {
        const int n_blk = static_cast<int>(t % args.num_n);
        const long long pt = t / args.num_n;
        const int img = static_cast<int>(pt / per_img);
        const int rem = static_cast<int>(pt - static_cast<long long>(img) * per_img);
        const int ty = rem / args.tiles_x, tx = rem - ty * args.tiles_x;
        int oy[2];
        bool valid[2];
        const int ox = tx * args.C + pcol;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            oy[h] = ty * args.R + prow + h;
            valid[h] = oy[h] < args.OH && ox < args.OW;
        }

        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        float raw[2][8];
        uint32_t fa1[4][4], fa2[4][4], fb1[4][4], fb2[4][4];  // two fragment sets: [k-step][a0..a3], hi / p1 and lo / p2
        int tap = 0, dy = 0, dx = 0;                          // tap of the k-block in `raw`
        ptx::mbar_wait_nocall(&hfull_bar[hb % kHaloStages], (hb / kHaloStages) & 1);
        gather(halo + (hb % kHaloStages) * hstage, 0, raw);

        auto step = [&](uint32_t (&f1)[4][4], uint32_t (&f2)[4][4], int kb) {
            split(raw, f1, f2);
            if (++tap == taps) {  // the box's last tap is in registers: hand the box back
                tap = dy = dx = 0;
                __syncwarp();
                ptx::mbar_arrive_if(&hempty_bar[hb % kHaloStages], lane == 0);
                ++hb;
            } else if (++dx == args.KW) {
                dx = 0;
                ++dy;
            }
            if (kb + 1 < kblocks) {
                if (tap == 0) ptx::mbar_wait_nocall(&hfull_bar[hb % kHaloStages], (hb / kHaloStages) & 1);
                gather(halo + (hb % kHaloStages) * hstage, dy * args.Cb + dx, raw);
            }
            const int stage = kbg % kStagesIg;
            ptx::mbar_wait_nocall(&full_bar[stage], (kbg / kStagesIg) & 1);
            const uint32_t b_base = ptx::smem_u32(smem + stage * kStage);
            ptx::wgmma_fence();
            if (BF) {
                const uint64_t dQ1 = make_smem_desc_none(b_base, 128, 512);
                const uint64_t dQ2 = make_smem_desc_none(b_base + kBTile, 128, 512);
#pragma unroll
                for (int kk = 0; kk < 2; ++kk) {
                    Wgmma<BN, 0>::mma(acc, f2[kk], dQ1 + 16 * kk, 1u);  // p2 * q1
                    Wgmma<BN, 0>::mma(acc, f1[kk], dQ2 + 16 * kk, 1u);  // p1 * q2
                    Wgmma<BN, 0>::mma(acc, f1[kk], dQ1 + 16 * kk, 1u);  // p1 * q1
                }
            } else {
                const uint64_t dB = make_smem_desc_sw128(b_base);
                const uint64_t dBlo = make_smem_desc_sw128(b_base + kBTile);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    if (PLANES == 2) {
                        Wgmma<BN, 1>::mma(acc, f2[kk], dB + 2 * kk, 1u);    // A_lo * B_hi
                        Wgmma<BN, 1>::mma(acc, f1[kk], dBlo + 2 * kk, 1u);  // A_hi * B_lo
                        Wgmma<BN, 1>::mma(acc, f1[kk], dB + 2 * kk, 1u);    // A_hi * B_hi
                    } else {
                        Wgmma<BN, 1>::mma(acc, f1[kk], dB + 2 * kk, 1u);
                    }
                }
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();  // k-block kb - 1 retired: its filter stage and fragment set are free
            __syncwarp();
            ptx::mbar_arrive_if(&empty_bar[(kbg + kStagesIg - 1) % kStagesIg], kb > 0 && lane == 0);
            ++kbg;
        };
        for (int kb = 0; kb < kblocks; kb += 2) {
            step(fa1, fa2, kb);
            if (kb + 1 < kblocks) step(fb1, fb2, kb + 1);
        }
        ptx::wgmma_wait<0>();
        __syncwarp();
        ptx::mbar_arrive_if(&empty_bar[(kbg - 1) % kStagesIg], lane == 0);
        halo_epilogue<BN>(acc, args, n_blk, img, oy, valid, ox, oplane, SH, SW, c, gq);
    }
}

// Pre-split halo kernel (BF16x3, switch igemm_presplit): the producer and the filter ring of conv_igemm_halo_kernel, but
// each 32-channel fp32 box is split ONCE, not once per tap.
//   split      = when a box lands, the 256 consumer threads convert it (split_bf16x2, the same bits as the per-tap split)
//                into two bf16 planes p1 / p2, [ch / 8][R + KH - 1 rows][C + KW - 1 columns][8 ch]: a pixel's 8 channels
//                are one 16-byte row.  The fp32 box goes back to the producer as soon as the conversion has read it; the
//                planes are double-buffered, so box b + 1 is converted (during the last k-block of box b, behind its
//                MMAs) while warps still read box b, and one named barrier of the consumers per box suffices.
//   A operand  = per k-block and warp 4 ldmatrix.x4 (2 k-steps x 2 planes): the 8 rows of each 8 x 8 matrix are
//                8 consecutive pixels of one patch row, so every tap (dy, dx) is the row address + (dy * pc + dx) * 16
//                bytes, 16-byte aligned and free of bank conflicts.  ldmatrix yields the m16n8k16 A layout of wgmma.
//   tile       = the halo kernel's 128-pixel patch.  A 256-pixel tile (two m64 accumulators per warpgroup) would halve
//                the filter bytes per output where BN = 64, but a 288-thread CTA gets at most 168 registers per thread
//                and the second accumulator and fragment sets do not fit: ptxas then serialises the wgmma.
// Per k-block the wgmma sequence (p2*q1, p1*q2, p1*q1 per k-step), the operand values, the k order and BN are those of conv_igemm_halo_kernel<BN, 3>: the result is bit-identical to it.
template <int BN>
__global__ void __launch_bounds__(kThreadsIg, 1)
conv_igemm_presplit_kernel(const __grid_constant__ CUtensorMap tmX, const HaloArgs args) {
    constexpr int kBTile = BN * 32 * 2;
    constexpr int kStage = 2 * kBTile;
    constexpr int HS = kHaloStages;  // fp32 boxes in flight
    constexpr int kConsumers = kConsumerWarps * 32;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
    float* halo = reinterpret_cast<float*>(smem + kStagesIg * kStage);
    const int cstride = args.Rb * args.Cb;
    const int hstage = 32 * cstride;
    const int units = 4 * args.pr * args.pc;  // 16-byte rows per bf16 plane
    const uint32_t pbytes = 16u * static_cast<uint32_t>(units);
    // [buffer 2][p1, p2][units][16 B], then the box word offset of every unit
    const uint32_t planes = ptx::smem_u32(halo + HS * hstage);
    const int* utab = reinterpret_cast<const int*>(smem + kStagesIg * kStage + HS * hstage * 4 + 4 * pbytes);
    __shared__ uint64_t full_bar[kStagesIg];
    __shared__ uint64_t empty_bar[kStagesIg];
    __shared__ uint64_t hfull_bar[HS];
    __shared__ uint64_t hempty_bar[HS];

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int per_img = args.tiles_x * args.tiles_y;
    const int taps = args.taps, KW = args.KW;
    const int ncb = args.kblocks / taps;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStagesIg; ++s) {
            ptx::mbar_init(&full_bar[s], 1);
            ptx::mbar_init(&empty_bar[s], kConsumerWarps);
        }
        for (int s = 0; s < HS; ++s) {
            ptx::mbar_init(&hfull_bar[s], 1);
            ptx::mbar_init(&hempty_bar[s], kConsumerWarps);
        }
        ptx::fence_barrier_init();
    }
    for (int u = threadIdx.x; u < units; u += kThreadsIg) {
        const int ch8 = u / (args.pr * args.pc), rem = u - ch8 * args.pr * args.pc;
        const int row = rem / args.pc, col = rem - row * args.pc;
        const_cast<int*>(utab)[u] = 8 * ch8 * cstride + row * args.Cb + col + args.xshift;
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        if (lane == 0)
            halo_producer<BN, 3, HS>(&tmX, nullptr, nullptr, args, smem, halo, hstage, full_bar, empty_bar, hfull_bar,
                                     hempty_bar);
        return;
    }

    // ===================== consumers =====================
    const int gq = lane >> 2, c = lane & 3;
    const int wcols = args.C >> 3;
    const int wy = warp / wcols, wx = warp - wy * wcols;
    const int prow = 2 * wy, pcol = 8 * wx + gq;     // this thread's pixels in each patch: rows prow + h, column pcol
    // ldmatrix row of this lane: matrix lane / 8 = (channels 8-15 of the k-step) * 2 + (pixel row prow + 1), its row
    // lane % 8 = patch column 8 * wx + lane % 8
    const int lm = lane >> 3;
    const uint32_t lrow = planes + 16u * static_cast<uint32_t>(((lm >> 1) * args.pr + prow + (lm & 1)) * args.pc + 8 * wx + (lane & 7));
    const uint32_t kstep_bytes = pbytes / 2;                                   // channels 16-31 of the block

    int hb = 0;   // boxes converted
    int kbg = 0;  // filter stages consumed
    // split box hb into plane buffer hb & 1 and hand the fp32 box back
    auto convert_next = [&]() {
        const int hs = hb % HS;
        ptx::mbar_wait_nocall(&hfull_bar[hs], (hb / HS) & 1);
        const float* box = halo + hs * hstage;
        const uint32_t dst = planes + static_cast<uint32_t>(hb & 1) * 2u * pbytes;
        for (int u = threadIdx.x; u < units; u += kConsumers) {
            const float* s = box + utab[u];
            float x[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) x[i] = s[i * cstride];
            uint32_t p1[4], p2[4];
#pragma unroll
            for (int w = 0; w < 4; ++w) split_bf16x2(x[2 * w], x[2 * w + 1], p1[w], p2[w]);
            ptx::st_shared_v4(dst + 16u * u, p1);
            ptx::st_shared_v4(dst + pbytes + 16u * u, p2);
        }
        __syncwarp();
        ptx::mbar_arrive_if(&hempty_bar[hs], lane == 0);
        ++hb;
    };

    const int oplane = args.OH * args.OW;
    const int SH = (args.OH + 1) >> 1, SW = (args.OW + 1) >> 1;
    convert_next();  // grid <= tiles: every CTA has a first box
    for (long long t = blockIdx.x; t < args.tiles; t += gridDim.x) {
        const int n_blk = static_cast<int>(t % args.num_n);
        const long long pt = t / args.num_n;
        const int img = static_cast<int>(pt / per_img);
        const int rem = static_cast<int>(pt - static_cast<long long>(img) * per_img);
        const int ty = rem / args.tiles_x, tx = rem - ty * args.tiles_x;
        const bool more_tiles = t + gridDim.x < args.tiles;
        const int kbg0 = kbg;

        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        uint32_t fa1[2][4], fa2[2][4], fb1[2][4], fb2[2][4], fc1[2][4], fc2[2][4];  // fragment sets: [k-step][a0..a3], p1 / p2
        uint32_t abuf = 0, toff = 0;  // ldmatrix row of the current box's buffer, byte offset of the current tap
        int dx = 0;

        // one k-block: fragments by ldmatrix, then the MMAs; `last` = the box's last k-block, behind whose MMAs the next
        // box is split (when there is one)
        auto step = [&](uint32_t (&f1)[2][4], uint32_t (&f2)[2][4], bool last, bool next) {
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                const uint32_t a = abuf + toff + kk * kstep_bytes;
                ptx::ldsm_x4(a, f1[kk]);
                ptx::ldsm_x4(a + pbytes, f2[kk]);
            }
            toff += 16;
            if (++dx == KW) {
                dx = 0;
                toff += 16u * static_cast<uint32_t>(args.pc - KW);
            }
            const int stage = kbg & (kStagesIg - 1);
            ptx::mbar_wait_nocall(&full_bar[stage], (kbg / kStagesIg) & 1);
            const uint32_t b_base = ptx::smem_u32(smem) + stage * kStage;
            ptx::wgmma_fence();
            const uint64_t dQ1 = make_smem_desc_none(b_base, 128, 512);
            const uint64_t dQ2 = make_smem_desc_none(b_base + kBTile, 128, 512);
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                Wgmma<BN, 0>::mma(acc, f2[kk], dQ1 + 16 * kk, 1u);  // p2 * q1
                Wgmma<BN, 0>::mma(acc, f1[kk], dQ2 + 16 * kk, 1u);  // p1 * q2
                Wgmma<BN, 0>::mma(acc, f1[kk], dQ1 + 16 * kk, 1u);  // p1 * q1
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();  // k-block kbg - 1 retired: its filter stage and fragment set are free
            if (last && next) convert_next();
            __syncwarp();
            ptx::mbar_arrive_if(&empty_bar[(kbg + kStagesIg - 1) & (kStagesIg - 1)], kbg != kbg0 && lane == 0);
            ++kbg;
        };
        for (int cb = 0; cb < ncb; ++cb) {
            ptx::named_bar_sync(1, kConsumers);  // every consumer has split this box and left the buffer it overwrote
            abuf = lrow + static_cast<uint32_t>((hb - 1) & 1) * 2u * pbytes;
            toff = 0;
            dx = 0;
            const bool next = cb + 1 < ncb || more_tiles;
            // fragment sets a, b alternate; an odd box ends on set c, so the next box starts on a free set a either way
            int i = 0;
            for (; i + 2 < taps; i += 2) {
                step(fa1, fa2, false, false);
                step(fb1, fb2, false, false);
            }
            if (i + 1 < taps) {
                step(fa1, fa2, false, false);
                step(fb1, fb2, true, next);
            } else {
                step(fc1, fc2, true, next);
            }
        }
        ptx::wgmma_wait<0>();
        __syncwarp();
        ptx::mbar_arrive_if(&empty_bar[(kbg - 1) & (kStagesIg - 1)], lane == 0);

        const int ox = tx * args.C + pcol;
        int oy[2];
        bool valid[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            oy[h] = ty * args.R + prow + h;
            valid[h] = oy[h] < args.OH && ox < args.OW;
        }
        halo_epilogue<BN>(acc, args, n_blk, img, oy, valid, ox, oplane, SH, SW, c, gq);
    }
}

// Bank model of one ld.shared of the halo gather: lane l reads column l / 4 of channel plane (l % 4) * (2 for the bf16
// pairs, 1 for tf32); the warp is conflict-free when its 32 words fall in 32 different banks (the starting column and
// row only rotate the pattern).
static bool halo_banks_conflict_free(int cstride, bool bf) {
    unsigned used = 0;
    for (int l = 0; l < 32; ++l) used |= 1u << (((l >> 2) + (bf ? 2 : 1) * (l & 3) * cstride) & 31);
    return used == 0xFFFFFFFFu;
}

static int halo_smem_bytes(int OC, int planes, int Rb, int Cb) {
    const int npl = planes == 3 ? 2 : planes;
    const int b_stage = npl * igemm_bn_for(OC) * 32 * (planes == 3 ? 2 : 4);
    return kStagesIg * b_stage + kHaloStages * 32 * Rb * Cb * 4 + 1024;
}

// Patch and box of the halo kernel for a layer, or false when the layer keeps conv_igemm_kernel.  Among the patches
// 16x8, 32x4, 8x16 and 64x2 (columns x rows) the one that computes the fewest padded pixels wins (earlier on a tie:
// smaller halo).
static bool halo_geometry(const IgemmProblem& p, HaloGeom& g) {
    if (p.stride_h != 1 || p.stride_w != 1 || p.dil_h > 1 || p.dil_w > 1 || p.IC % 32 != 0) return false;
    const int taps = p.KH * p.KW;
    if (taps < 2 || taps > 63 || p.W % 4 != 0 || p.OH < 1 || p.OW < 1) return false;  // 1x1: no tap reuse
    if (p.input != nullptr && (reinterpret_cast<uintptr_t>(p.input) & 15) != 0) return false;  // TMA: 16-byte base
    static const int kCols[4] = {16, 32, 8, 64};
    long long best = -1;
    for (int C : kCols) {
        const int R = 128 / C;
        const long long cost = static_cast<long long>(ceil_div(p.OW, C)) * C * ceil_div(p.OH, R) * R;
        const int xshift = ((p.pad_left + 3) & ~3) - p.pad_left;
        const int rb0 = R + p.KH - 1, cb0 = (C + p.KW - 1 + xshift + 3) & ~3;  // 16-byte box rows
        int rb = 0, cbx = 0;
        for (int dc = 0; dc <= 12; dc += 4)
            for (int dr = 0; dr < 8; ++dr) {
                const int r = rb0 + dr, cc = cb0 + dc;
                if (r > 256 || cc > 256 || !halo_banks_conflict_free(r * cc, p.planes == 3)) continue;
                if (rb == 0 || r * cc < rb * cbx) { rb = r; cbx = cc; }
            }
        if (rb == 0 || halo_smem_bytes(p.OC, p.planes, rb, cbx) > 227 * 1024) continue;
        if (best < 0 || cost < best) {
            best = cost;
            g.R = R; g.C = C; g.Rb = rb; g.Cb = cbx;
        }
    }
    return best >= 0;
}

// Box of conv_igemm_presplit_kernel for a layer the halo kernel takes in BF16x3 mode, or false (the layer keeps the
// halo kernel).  The patch is the halo kernel's; the box is the patch plus its halo, unpadded: the split reads it along
// rows, free of bank conflicts at any plane stride.
static int presplit_smem_bytes(int OC, int Rb, int Cb, int pr, int pc) {
    const int units = 4 * pr * pc;
    return kStagesIg * 2 * igemm_bn_for(OC) * 64 + kHaloStages * 32 * Rb * Cb * 4 + 2 * 32 * units + 4 * units + 1024;
}

static bool presplit_geometry(const IgemmProblem& p, HaloGeom& g) {
    HaloGeom h;
    if (p.planes != 3 || !halo_geometry(p, h)) return false;
    const int xshift = ((p.pad_left + 3) & ~3) - p.pad_left;
    g.R = h.R; g.C = h.C;
    g.Rb = h.R + p.KH - 1;
    g.Cb = (h.C + p.KW - 1 + xshift + 3) & ~3;
    return presplit_smem_bytes(p.OC, g.Rb, g.Cb, g.Rb, h.C + p.KW - 1) <= 227 * 1024;
}

// The input blob [N][in_img_c][H][W] (the IC channels of this slice) in boxes of hg.Cb x hg.Rb x 32 channels; boxes past
// its edges read as zeros
static int halo_input_map(const IgemmProblem& p, const HaloGeom& hg, EncodeTiledFn enc, CUtensorMap* tmX) {
    const cuuint64_t in_c = static_cast<cuuint64_t>(p.in_c_total > 0 ? p.in_c_total : p.IC);
    cuuint64_t dims[4] = {(cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.IC, (cuuint64_t)p.N};
    cuuint64_t strides[3] = {(cuuint64_t)p.W * 4, (cuuint64_t)p.W * p.H * 4, in_c * p.H * p.W * 4};
    cuuint32_t box[4] = {(cuuint32_t)hg.Cb, (cuuint32_t)hg.Rb, 32, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(tmX, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(p.input), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "fcuda: igemm input tensor map failed (%d)\n", (int)r);
        return FCUDA_ERR_CUDA;
    }
    return 0;
}

static HaloArgs halo_args(const IgemmProblem& p, const HaloGeom& hg, int BN) {
    const int taps = p.KH * p.KW;
    HaloArgs a;
    a.residual = p.residual; a.out = p.output; a.bias = p.bias;
    a.OC = p.OC; a.OH = p.OH; a.OW = p.OW; a.KW = p.KW; a.taps = taps;
    a.out_img_c = p.out_c_total > 0 ? p.out_c_total : p.OC;
    a.kblocks = ceil_div(taps * p.IC, 32);
    a.num_n = ceil_div(p.OC, BN);
    a.relu = p.relu;
    a.pool = p.pool ? 1 : 0;
    a.R = hg.R; a.C = hg.C;
    a.tiles_x = ceil_div(p.OW, hg.C);
    a.tiles_y = ceil_div(p.OH, hg.R);
    a.Rb = hg.Rb; a.Cb = hg.Cb;
    a.pad_top = p.pad_top;
    a.xpad = (p.pad_left + 3) & ~3;
    a.xshift = a.xpad - p.pad_left;
    a.tiles = static_cast<long long>(p.N) * a.tiles_x * a.tiles_y * a.num_n;
    a.wbf = reinterpret_cast<const unsigned char*>(p.w_hi);
    a.wbf_kb_bytes = 2u * static_cast<unsigned>(igemm_ocpad(p.OC)) * 64u;
    a.pr = hg.R + p.KH - 1;
    a.pc = hg.C + p.KW - 1;
    return a;
}

template <int BN>
int launch_igemm_presplit(const IgemmProblem& p, const HaloGeom& hg, cudaStream_t stream) {
    EncodeTiledFn enc = encode_fn();
    if (!enc) return FCUDA_ERR_CUDA;
    CUtensorMap tmX;
    if (int rc = halo_input_map(p, hg, enc, &tmX)) return rc;
    const int taps = p.KH * p.KW;
    if (igemm_bn_for(p.OC) != BN || static_cast<unsigned long long>(ceil_div(taps * p.IC, 32)) * igemm_ocpad(p.OC) * 128ull >= (1ull << 31))
        return -1;
    HaloArgs a = halo_args(p, hg, BN);
    const long long pixel_tiles = a.tiles / a.num_n;
    if (static_cast<long long>(p.OH) * p.OW >= (1ll << 30) || a.tiles * a.kblocks >= (1ll << 31)) return -1;
    const int smem = presplit_smem_bytes(p.OC, hg.Rb, hg.Cb, a.pr, a.pc);
    auto kern = conv_igemm_presplit_kernel<BN>;
    static SmemAttrCache attr_cache;
    if (int rc = ensure_dynamic_smem(kern, smem, attr_cache)) return rc;
    int per_sm = 0;
    FCUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreadsIg, smem));
    const long long slots = static_cast<long long>(sm_count()) * (per_sm > 0 ? per_sm : 1);
    const unsigned grid = static_cast<unsigned>(a.tiles < slots ? a.tiles : slots);
    const double macs = static_cast<double>(p.N) * p.OC * p.OH * p.OW * p.IC * taps;
    const double mma = 2.0 * static_cast<double>(pixel_tiles) * hg.R * hg.C * (a.num_n * BN) * (a.kblocks * 32) * 3;
    const int prof = prof_begin(stream, PROF_IGEMM, 2.0 * macs, mma,
                                4.0 * (static_cast<double>(p.N) * p.IC * p.H * p.W + static_cast<double>(p.OC) * taps * p.IC +
                                       static_cast<double>(p.N) * p.OC * p.OH * p.OW * (p.residual ? 2 : 1)));
    kern<<<grid, kThreadsIg, smem, stream>>>(tmX, a);
    prof_end(prof, stream);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

template <int BN, int PLANES>
int launch_igemm_halo(const IgemmProblem& p, const HaloGeom& hg, cudaStream_t stream) {
    constexpr bool BF = PLANES == 3;
    constexpr int NPL = BF ? 2 : PLANES;
    const int taps = p.KH * p.KW;
    const int K = taps * p.IC;
    EncodeTiledFn enc = encode_fn();
    if (!enc) return FCUDA_ERR_CUDA;
    CUtensorMap tmX, tmW, tmWlo;
    memset(&tmW, 0, sizeof(tmW));
    tmWlo = tmW;
    if (!BF) {
        const int Kf = (K + 3) & ~3;
        for (int pl = 0; pl < NPL; ++pl) {
            cuuint64_t dims[3] = {(cuuint64_t)Kf, (cuuint64_t)p.OC, 1};
            cuuint64_t strides[2] = {(cuuint64_t)Kf * 4, (cuuint64_t)Kf * p.OC * 4};
            cuuint32_t box[3] = {32, (cuuint32_t)BN, 1};
            cuuint32_t estr[3] = {1, 1, 1};
            const float* base = pl == 0 ? p.w_hi : p.w_lo;
            CUresult r = enc(pl == 0 ? &tmW : &tmWlo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides,
                             box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
                fprintf(stderr, "fcuda: igemm weight tensor map failed (%d)\n", (int)r);
                return FCUDA_ERR_CUDA;
            }
        }
    }
    if (int rc = halo_input_map(p, hg, enc, &tmX)) return rc;
    if (BF && (igemm_bn_for(p.OC) != BN || static_cast<unsigned long long>(ceil_div(K, 32)) * igemm_ocpad(p.OC) * 128ull >= (1ull << 31))) return -1;
    HaloArgs a = halo_args(p, hg, BN);
    const long long pixel_tiles = a.tiles / a.num_n;
    if (static_cast<long long>(p.OH) * p.OW >= (1ll << 30) || a.tiles * a.kblocks >= (1ll << 31)) return -1;
    const int smem = halo_smem_bytes(p.OC, PLANES, hg.Rb, hg.Cb);
    auto kern = conv_igemm_halo_kernel<BN, PLANES>;
    static SmemAttrCache attr_cache;
    if (int rc = ensure_dynamic_smem(kern, smem, attr_cache)) return rc;
    int per_sm = 0;
    FCUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreadsIg, smem));
    const long long slots = static_cast<long long>(sm_count()) * (per_sm > 0 ? per_sm : 1);
    const unsigned grid = static_cast<unsigned>(a.tiles < slots ? a.tiles : slots);
    // the same algorithmic work as conv_igemm_kernel; the issued MMA work includes the padded patch pixels
    const double macs = static_cast<double>(p.N) * p.OC * p.OH * p.OW * p.IC * taps;
    const double mma = 2.0 * static_cast<double>(pixel_tiles) * 128 * (a.num_n * BN) * (a.kblocks * 32) * (PLANES >= 2 ? 3 : 1);
    const int prof = prof_begin(stream, PROF_IGEMM, 2.0 * macs, mma,
                                4.0 * (static_cast<double>(p.N) * p.IC * p.H * p.W + static_cast<double>(p.OC) * K +
                                       static_cast<double>(p.N) * p.OC * p.OH * p.OW * (p.residual ? 2 : 1)));
    kern<<<grid, kThreadsIg, smem, stream>>>(tmX, tmW, tmWlo, a);
    prof_end(prof, stream);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace

bool conv_igemm_halo_geometry(const IgemmProblem& p, HaloGeom* g) {
    HaloGeom tmp;
    const bool ok = halo_geometry(p, tmp);
    if (ok && g) *g = tmp;
    return ok;
}

bool conv_igemm_presplit_geometry(const IgemmProblem& p, HaloGeom* g) {
    HaloGeom tmp;
    const bool ok = presplit_geometry(p, tmp);
    if (ok && g) *g = tmp;
    return ok;
}

bool conv_igemm_supported(int IC, int KH, int KW) {
    if (KH * KW > 63) return false;                               // per-pixel tap validity mask is 64-bit
    if (IC % 32 != 0 && KH * KW * IC > kMaxTableK) return false;  // k-table must fit in shared memory
    return true;
}

size_t conv_igemm_packed_floats(int OC, int IC, int taps, int planes) {
    const size_t rows = static_cast<size_t>(planes) * OC * ((taps * IC + 3) & ~3);
    if (planes < 2) return rows;
    // the pre-tiled BF16x3 planes (2 planes x k-blocks x OCpad x 64 bytes) must fit the same buffer
    const size_t tiled = (2 * static_cast<size_t>(ceil_div(taps * IC, 32)) * igemm_ocpad(OC) * 64 + 3) / 4;
    return rows > tiled ? rows : tiled;
}

int conv_igemm_pack_weights(const float* w, float* w_hi, float* w_lo, int OC, int IC, int taps, cudaStream_t s, int bf16x3) {
    if (bf16x3) {
        const int KB = ceil_div(taps * IC, 32), OCpad = igemm_ocpad(OC);
        const size_t total8 = static_cast<size_t>(KB) * OCpad * 32;
        igemm_pack_weights_bf16_kernel<<<static_cast<unsigned>(ceil_div_sz(total8, 256)), 256, 0, s>>>(
            w, reinterpret_cast<__nv_bfloat16*>(w_hi), OC, IC, taps, KB, OCpad, igemm_bn_for(OC));
        FCUDA_CHECK_LAUNCH();
        count_launch();
        return 0;
    }
    const int Kf = (taps * IC + 3) & ~3;
    const size_t total = static_cast<size_t>(OC) * Kf;
    igemm_pack_weights_kernel<<<static_cast<unsigned>(ceil_div_sz(total, 256)), 256, 0, s>>>(w, w_hi, w_lo, OC, IC, taps, Kf);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

// The fused 2x2 max pooling serves the 3x3 / stride-1 layers with whole 32-channel blocks that precede a pooling layer
// (VGG-style stacks); the other layers keep a separate pooling launch.
bool conv_igemm_can_pool(const IgemmProblem& p) {
    return p.KH == 3 && p.KW == 3 && p.stride_h == 1 && p.stride_w == 1 && p.dil_h <= 1 && p.dil_w <= 1 && p.IC % 32 == 0 &&
           p.pad_top <= 2 && p.pad_left <= 2 && p.W % 4 == 0 && p.residual == nullptr &&
           (p.input == nullptr || (reinterpret_cast<uintptr_t>(p.input) & 15) == 0);
}

int conv_igemm_forward(const IgemmProblem& p, cudaStream_t stream) {
    if (!conv_igemm_supported(p.IC, p.KH, p.KW)) return -1;
    if (p.pool && !conv_igemm_can_pool(p)) return -200;
    const int bn = igemm_bn_for(p.OC);
    HaloGeom hg;
    if (tune_get(TUNE_IGEMM_HALO) != 0 && halo_geometry(p, hg)) {
        HaloGeom pg;
        if (p.planes == 3 && tune_get(TUNE_IGEMM_PRESPLIT) != 0 && presplit_geometry(p, pg))
            return bn == 32 ? launch_igemm_presplit<32>(p, pg, stream) : bn == 64 ? launch_igemm_presplit<64>(p, pg, stream) : launch_igemm_presplit<128>(p, pg, stream);
        if (p.planes == 3) return bn == 32 ? launch_igemm_halo<32, 3>(p, hg, stream) : bn == 64 ? launch_igemm_halo<64, 3>(p, hg, stream) : launch_igemm_halo<128, 3>(p, hg, stream);
        if (p.planes == 2) return bn == 32 ? launch_igemm_halo<32, 2>(p, hg, stream) : bn == 64 ? launch_igemm_halo<64, 2>(p, hg, stream) : launch_igemm_halo<128, 2>(p, hg, stream);
        return bn == 32 ? launch_igemm_halo<32, 1>(p, hg, stream) : bn == 64 ? launch_igemm_halo<64, 1>(p, hg, stream) : launch_igemm_halo<128, 1>(p, hg, stream);
    }
    if (p.planes == 3) return bn == 32 ? launch_igemm<32, 3>(p, stream) : bn == 64 ? launch_igemm<64, 3>(p, stream) : launch_igemm<128, 3>(p, stream);
    if (p.planes == 2) return bn == 32 ? launch_igemm<32, 2>(p, stream) : bn == 64 ? launch_igemm<64, 2>(p, stream) : launch_igemm<128, 2>(p, stream);
    return bn == 32 ? launch_igemm<32, 1>(p, stream) : bn == 64 ? launch_igemm<64, 1>(p, stream) : launch_igemm<128, 1>(p, stream);
}

}  // namespace fcuda
