// Winograd F(6,3) and F(2,3) transform kernels (sm_90a).
//
// Replaces, on the GPU:
//   transformKernel_F6x6_3x3           /root/reference/src/booster/avx/winograd_kernels_F63.cpp:222-271   (filter, at Init)
//   pad_input + winogradInputFrameTransformSeq   generic_kernels.cpp:31-48, winograd_kernels_F63.cpp:272-513
//   winogradOutputTransform<RELU,BIAS>           winograd_kernels_F63.cpp:1029-1269
//   F(2,3) variant                     /root/reference/src/booster/arm/winograd_kernels.cpp:115-279 (NEON only upstream)
// The 64 (16) per-tile-element GEMMs in between run on wgmma (tensor_gemm.cu).
//
// Layouts (private to this backend — parity is defined on NCHW blobs only, SURVEY.md §8):
//   U[e][oc][ic]   transformed filters, K-major rows for the TensorGEMM B operand
//   V[e][t][ic]    transformed input tiles, t = chunk-local tile index, K-major rows for the A operand (plain fp32:
//                  the TensorGEMM makes the TF32 hi/lo split on chip)
//   M[e][t][oc]    products
// U exists as a TF32-exact "hi" plane and (3xTF32 mode) an fp32-remainder "lo" plane.
//
// Data movement: a block stages a (32 channels) x (8 rows) x (5 tiles wide) slab through shared memory so that
// global reads are coalesced along x and global writes are coalesced along the channel (K) dimension;
// zero padding is applied by the bounds check of the slab load (no padded copy of the input is made).
#include "winograd.cuh"
#include "common.cuh"

namespace fcuda {

// ------------------------------------------------------------------------------------------------
// 1-D transforms
// ------------------------------------------------------------------------------------------------
// B^T for F(6,3): same constants and operation order as winograd_kernels_F63.cpp:297-321.
__device__ __forceinline__ void f63_bt(const float (&r)[8], float (&o)[8]) {
    o[0] = (r[0] - r[6]) + (r[4] - r[2]) * 5.25f;
    o[7] = (r[7] - r[1]) + (r[3] - r[5]) * 5.25f;
    const float t1 = (r[2] + r[6]) - r[4] * 4.25f;
    const float t2 = (r[1] + r[5]) - r[3] * 4.25f;
    const float s1 = r[4] * 1.25f;
    const float s2 = r[3] * 2.5f;
    float p1 = r[6] + (r[2] * 0.25f - s1);
    float p2 = (r[1] * 0.5f - s2) + r[5] * 2.f;
    o[3] = p1 + p2;
    o[4] = p1 - p2;
    p1 = r[6] + (r[2] - s1) * 4.f;
    p2 = (r[1] * 2.f - s2) + r[5] * 0.5f;
    o[5] = p1 + p2;
    o[6] = p1 - p2;
    o[1] = t1 + t2;
    o[2] = t1 - t2;
}

// A^T for F(6,3): winograd_kernels_F63.cpp:1040-1045.
__device__ __forceinline__ void f63_at(const float (&m)[8], float (&s)[6]) {
    const float a12 = m[1] + m[2], s12 = m[1] - m[2];
    const float a34 = m[3] + m[4], s34 = m[3] - m[4];
    const float a56 = m[5] + m[6], s56 = m[5] - m[6];
    s[0] = m[0] + a12 + a34 + 32.f * a56;
    s[1] = s12 + 2.f * s34 + 16.f * s56;
    s[2] = a12 + 4.f * a34 + 8.f * a56;
    s[3] = s12 + 8.f * s34 + 4.f * s56;
    s[4] = a12 + 16.f * a34 + 2.f * a56;
    s[5] = s12 + 32.f * s34 + s56 + m[7];
}

// F(2,3): B^T = [1 0 -1 0; 0 1 1 0; 0 -1 1 0; 0 1 0 -1], A^T = [1 1 1 0; 0 1 -1 -1]
__device__ __forceinline__ void f23_bt(const float (&r)[4], float (&o)[4]) {
    o[0] = r[0] - r[2];
    o[1] = r[1] + r[2];
    o[2] = r[2] - r[1];
    o[3] = r[1] - r[3];
}
__device__ __forceinline__ void f23_at(const float (&m)[4], float (&s)[2]) {
    s[0] = m[0] + m[1] + m[2];
    s[1] = m[1] - m[2] - m[3];
}

template <int T> struct Wino;  // T = input tile edge
template <> struct Wino<8> {
    static constexpr int kIn = 8, kOut = 6;
    __device__ static __forceinline__ void bt(const float (&r)[8], float (&o)[8]) { f63_bt(r, o); }
    __device__ static __forceinline__ void at(const float (&m)[8], float (&s)[6]) { f63_at(m, s); }
};
template <> struct Wino<4> {
    static constexpr int kIn = 4, kOut = 2;
    __device__ static __forceinline__ void bt(const float (&r)[4], float (&o)[4]) { f23_bt(r, o); }
    __device__ static __forceinline__ void at(const float (&m)[4], float (&s)[2]) { f23_at(m, s); }
};

// ------------------------------------------------------------------------------------------------
// Filter transform  U = G g G^T   (Init time)
// ------------------------------------------------------------------------------------------------
// G for F(6,3): the reference's table, winograd_kernels_F63.cpp:191-201 (rows 5/6 pre-divided by 32 to match
// the x32 in the output transform).
__constant__ float kG63[8][3] = {
    {1.0f, 0.0f, 0.0f},
    {-2.0f / 9, -2.0f / 9, -2.0f / 9},
    {-2.0f / 9, 2.0f / 9, -2.0f / 9},
    {1.0f / 90, 1.0f / 45, 2.0f / 45},
    {1.0f / 90, -1.0f / 45, 2.0f / 45},
    {1.0f / 45, 1.0f / 90, 1.0f / 180},
    {1.0f / 45, -1.0f / 90, 1.0f / 180},
    {0.0f, 0.0f, 1.0f}};
__constant__ float kG23[4][3] = {{1.f, 0.f, 0.f}, {0.5f, 0.5f, 0.5f}, {0.5f, -0.5f, 0.5f}, {0.f, 0.f, 1.f}};

template <int T>
__device__ __forceinline__ float wino_G(int i, int k) {
    if constexpr (T == 8) return kG63[i][k];
    else return kG23[i][k];
}

template <int T>
__global__ void __launch_bounds__(128)
wino_filter_kernel(const float* __restrict__ w, float* __restrict__ U_hi, float* __restrict__ U_lo, int OC, int IC) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // oc * IC + ic
    if (idx >= OC * IC) return;
    const int oc = idx / IC, ic = idx - oc * IC;
    float g[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) g[i] = w[static_cast<size_t>(idx) * 9 + i];
    float mid[T][3];
#pragma unroll
    for (int i = 0; i < T; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 3; ++k) s += wino_G<T>(i, k) * g[k * 3 + j];
            mid[i][j] = s;
        }
#pragma unroll
    for (int i = 0; i < T; ++i)
#pragma unroll
        for (int j = 0; j < T; ++j) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 3; ++k) s += mid[i][k] * wino_G<T>(j, k);
            const size_t o = (static_cast<size_t>(i * T + j) * OC + oc) * IC + ic;
            if (U_lo) {
                float hi, lo;
                split_tf32(s, hi, lo);
                U_hi[o] = hi;
                U_lo[o] = lo;
            } else {
                U_hi[o] = s;
            }
        }
}

// ------------------------------------------------------------------------------------------------
// Input transform  V = B^T d B
// ------------------------------------------------------------------------------------------------
// Both transform kernels are issue-bound if written naively (first version: 3.4k instructions per thread, 60% of
// them index arithmetic of a flat slab loop), so the block shape is chosen to make the data movement trivially
// addressable: 5 tiles per block => an input slab row is exactly 32 floats (5*6+2) — one warp request per
// (channel,row) line — and an output slab row is 30 floats.  One warp per tile, one lane per channel.
constexpr int kSegTiles = 5;   // tiles per block along x (one warp each)
constexpr int kChBlock = 32;   // channels per block (one lane each)
constexpr int kXformThreads = kSegTiles * 32;

// 4-byte asynchronous global -> shared copy (LDGSTS); ok == false writes a zero without touching global memory
__device__ __forceinline__ void cp_async4_zfill(float* smem_dst, const float* gmem_src, bool ok) {
    const unsigned sz = ok ? 4u : 0u;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;"
                 ::"r"(static_cast<unsigned>(__cvta_generic_to_shared(smem_dst))), "l"(gmem_src), "r"(sz)
                 : "memory");
}

template <int T>
__global__ void __launch_bounds__(kXformThreads)
wino_input_kernel(const float* __restrict__ in, float* __restrict__ V, WinoGeom g, int R0, int Tc, int ncb) {
    using W = Wino<T>;
    constexpr int OT = W::kOut;
    constexpr int COLS = OT * kSegTiles + (T - OT);  // 32 for F(6,3)
    constexpr int CH_STRIDE = T * COLS + 1;          // odd => conflict-free when lanes index channels
    __shared__ float slab[kChBlock * CH_STRIDE];

    // ncb > 0: 1-D grid with the channel block as the FASTEST index — the blocks that write the eight 128-byte pieces of the
    // same 1 KB row V[e][tile][0..IC) run at the same time, so DRAM sees whole rows instead of 128 B at a 1 KB stride
    const int segs = (g.tilesX + kSegTiles - 1) / kSegTiles;
    const unsigned bx = ncb > 0 ? blockIdx.x / static_cast<unsigned>(ncb) : blockIdx.x;
    const int seg = bx % segs;
    const int Rl = bx / segs;  // chunk-local tile-row
    const int R = R0 + Rl;
    const int n = R / g.tilesY, ty = R - n * g.tilesY;
    const int tx0 = seg * kSegTiles;
    const int c0 = (ncb > 0 ? blockIdx.x % static_cast<unsigned>(ncb) : blockIdx.y) * kChBlock;
    const int gy0 = ty * OT - g.pad_top, gx0 = tx0 * OT - g.pad_left;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // Slab load: warp w takes channels w, w+5, ...; lane = column.  Every line of the slab is an asynchronous 4-byte
    // copy: all ~52 loads of a lane are in flight at once (one memory latency per block), no staging registers, no STS;
    // padding = zero-fill copies that do not touch global memory.
    {
        const size_t plane = static_cast<size_t>(g.H) * g.W;
        const float* img = in + static_cast<size_t>(n) * g.C_in * plane;
        const int gx = gx0 + lane;
        const bool x_ok = lane < COLS && gx >= 0 && gx < g.W;
        unsigned row_ok = 0;
#pragma unroll
        for (int r = 0; r < T; ++r)
            if (static_cast<unsigned>(gy0 + r) < static_cast<unsigned>(g.H)) row_ok |= 1u << r;
        if (lane < COLS) {
            for (int c = w; c < kChBlock; c += kSegTiles) {
                const int ic = c0 + c;
                const bool c_ok = x_ok && ic < g.C_in;
                const float* p = c_ok ? img + static_cast<size_t>(ic) * plane + static_cast<long long>(gy0) * g.W + gx : in;
                float* sp = slab + c * CH_STRIDE + lane;
#pragma unroll
                for (int r = 0; r < T; ++r) {
                    const bool ok = c_ok && ((row_ok >> r) & 1u);
                    cp_async4_zfill(sp + r * COLS, ok ? p + r * g.W : in, ok);
                }
            }
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
    }
    __syncthreads();

    const int tx = tx0 + w, ic = c0 + lane;
    if (tx >= g.tilesX || ic >= g.C_in) return;
    const float* d = slab + lane * CH_STRIDE + w * OT;

    float t[T][T];
#pragma unroll
    for (int x = 0; x < T; ++x) {
        float col[T], o[T];
#pragma unroll
        for (int y = 0; y < T; ++y) col[y] = d[y * COLS + x];
        W::bt(col, o);
#pragma unroll
        for (int y = 0; y < T; ++y) t[y][x] = o[y];
    }
    const size_t tp = static_cast<size_t>(Rl) * g.tilesX + tx;  // chunk-local tile index
    // bytes per tile element plane; < 2^32 because all T*T planes live in HBM together
    const uint32_t plane_bytes = static_cast<uint32_t>(Tc) * static_cast<uint32_t>(g.C_in) * 4u;
    char* vp = reinterpret_cast<char*>(V + tp * g.C_in + ic);  // plain fp32: the TensorGEMM splits hi/lo on chip
#pragma unroll
    for (int a = 0; a < T; ++a) {
        float o[T];
        W::bt(t[a], o);
#pragma unroll
        for (int b = 0; b < T; ++b)  // one IMAD.WIDE.U32 + STG per element
            *reinterpret_cast<float*>(vp + static_cast<unsigned long long>(plane_bytes) * static_cast<uint32_t>(a * T + b)) = o[b];
    }
}

// ------------------------------------------------------------------------------------------------
// Output transform  Y = A^T M A  (+bias, ReLU / Clip clamp), clipped NCHW store; POOL: a following 2x2 / stride-2 max pooling
// (pooling_layer.h:38-91, pad 0) is applied to the tile in registers — the 6x6 (2x2) output tile starts at an even
// coordinate, so no window straddles two tiles — and only the pooled (OH+1)/2 x (OW+1)/2 blob is written.
// ------------------------------------------------------------------------------------------------
template <int T, bool POOL, bool CLIP>
__global__ void __launch_bounds__(kXformThreads)
wino_output_kernel(const float* __restrict__ M, float* __restrict__ out, const float* __restrict__ bias, WinoGeom g,
                   int R0, int Tc, int act, float lo, float hi, int ncb) {
    using W = Wino<T>;
    constexpr int OT = W::kOut;
    constexpr int ST = POOL ? OT / 2 : OT;     // rows / columns of the tile as stored
    constexpr int COLS = ST * kSegTiles;       // 30 (15 pooled) for F(6,3)
    constexpr int CH_STRIDE = ST * COLS + 1;
    __shared__ float slab[kChBlock * CH_STRIDE];

    const int segs = (g.tilesX + kSegTiles - 1) / kSegTiles;
    const unsigned bx = ncb > 0 ? blockIdx.x / static_cast<unsigned>(ncb) : blockIdx.x;  // ncb > 0: channel block fastest (see above)
    const int seg = bx % segs;
    const int Rl = bx / segs;
    const int R = R0 + Rl;
    const int n = R / g.tilesY, ty = R - n * g.tilesY;
    const int tx0 = seg * kSegTiles;
    const int c0 = (ncb > 0 ? blockIdx.x % static_cast<unsigned>(ncb) : blockIdx.y) * kChBlock;

    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tx = tx0 + w, oc = c0 + lane;
    if (tx < g.tilesX && oc < g.C_out) {
        const size_t tp = static_cast<size_t>(Rl) * g.tilesX + tx;
        const uint32_t plane_bytes = static_cast<uint32_t>(Tc) * static_cast<uint32_t>(g.C_out) * 4u;
        const char* m = reinterpret_cast<const char*>(M + tp * g.C_out + oc);
        float mm[T][T];
#pragma unroll
        for (int a = 0; a < T; ++a)
#pragma unroll
            for (int b = 0; b < T; ++b)
                if (T == 8) {
                    // all T*T plane loads issued back to back (volatile: nvcc otherwise interleaves them column by column with
                    // the transform to save registers — 56 registers, eight dependent rounds of memory latency per tile)
                    asm volatile("ld.volatile.global.f32 %0, [%1];"
                                 : "=f"(mm[a][b])
                                 : "l"(m + static_cast<unsigned long long>(plane_bytes) * static_cast<uint32_t>(a * T + b)));
                } else {
                    mm[a][b] = __ldg(reinterpret_cast<const float*>(
                        m + static_cast<unsigned long long>(plane_bytes) * static_cast<uint32_t>(a * T + b)));
                }
        float tmp[OT][T];
#pragma unroll
        for (int b = 0; b < T; ++b) {
            float col[T], s[OT];
#pragma unroll
            for (int a = 0; a < T; ++a) col[a] = mm[a][b];
            W::at(col, s);
#pragma unroll
            for (int i = 0; i < OT; ++i) tmp[i][b] = s[i];
        }
        const float bv = bias ? __ldg(bias + oc) : 0.f;
        float* dst = slab + lane * CH_STRIDE + w * ST;
        if (!POOL) {
#pragma unroll
            for (int i = 0; i < OT; ++i) {
                float s[OT];
                W::at(tmp[i], s);
#pragma unroll
                for (int j = 0; j < OT; ++j) {
                    float v = s[j] + bv;
                    if (act) v = act_clamp<CLIP>(v, lo, hi);
                    dst[i * COLS + j] = v;
                }
            }
        } else {
            // outputs outside the image (partial tiles, odd OH / OW) must not win a window: -inf
            const int oy0 = ty * OT, ox0 = tx * OT;
#pragma unroll
            for (int i = 0; i < OT; i += 2) {
                float s0[OT], s1[OT];
                W::at(tmp[i], s0);
                W::at(tmp[i + 1], s1);
                const bool r1 = oy0 + i + 1 < g.OH;
#pragma unroll
                for (int j = 0; j < OT; j += 2) {
                    const bool c1 = ox0 + j + 1 < g.OW;
                    float v = s0[j];
                    if (c1) v = fmaxf(v, s0[j + 1]);
                    if (r1) {
                        v = fmaxf(v, s1[j]);
                        if (c1) v = fmaxf(v, s1[j + 1]);
                    }
                    v += bv;  // max commutes with the per-channel bias and with the clamp
                    if (act) v = act_clamp<CLIP>(v, lo, hi);
                    dst[(i >> 1) * COLS + (j >> 1)] = v;
                }
            }
        }
    }
    __syncthreads();

    // store: warp w takes channels w, w+5, ...; the ST rows of a channel are unrolled; lane = column
    const int SH = POOL ? (g.OH + 1) / 2 : g.OH, SW = POOL ? (g.OW + 1) / 2 : g.OW;  // stored blob geometry
    const int oy0 = ty * ST, ox = tx0 * ST + lane;
    const size_t oplane = static_cast<size_t>(SH) * SW;
    float* img = out + static_cast<size_t>(n) * g.C_out * oplane;
    const bool x_ok = lane < COLS && ox < SW;
    unsigned row_ok = 0;
#pragma unroll
    for (int r = 0; r < ST; ++r)
        if (oy0 + r < SH) row_ok |= 1u << r;
    for (int c = w; c < kChBlock; c += kSegTiles) {
        const int o = c0 + c;
        if (!(x_ok && o < g.C_out)) continue;
        float* p = img + static_cast<size_t>(o) * oplane + static_cast<size_t>(oy0) * SW + ox;
        const float* sp = slab + c * CH_STRIDE + lane;
#pragma unroll
        for (int r = 0; r < ST; ++r)
            if ((row_ok >> r) & 1u) p[r * SW] = sp[r * COLS];
    }
}

// ------------------------------------------------------------------------------------------------
// Host launchers
// ------------------------------------------------------------------------------------------------
int wino_filter_transform(int tile, const float* w, float* U_hi, float* U_lo, int OC, int IC, cudaStream_t s) {
    const int total = OC * IC;
    const int blocks = ceil_div(total, 128);
    if (tile == 8) wino_filter_kernel<8><<<blocks, 128, 0, s>>>(w, U_hi, U_lo, OC, IC);
    else wino_filter_kernel<4><<<blocks, 128, 0, s>>>(w, U_hi, U_lo, OC, IC);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

int wino_input_transform(int tile, const float* in, float* V, const WinoGeom& g, int R0, int R1, cudaStream_t s) {
    const int segs = ceil_div(g.tilesX, kSegTiles);
    const int Tc = (R1 - R0) * g.tilesX;
    dim3 grid(static_cast<unsigned>(segs) * (R1 - R0), ceil_div(g.C_in, kChBlock));
    int ncb = 0;
    if (static_cast<unsigned long long>(grid.x) * grid.y < 0x7fffffffULL) {
        ncb = static_cast<int>(grid.y);
        grid = dim3(grid.x * grid.y, 1);
    }
    // algorithmic bytes: the rows of the input the chunk covers, read once, + V written once
    const double imgs = static_cast<double>(R1 - R0) / g.tilesY;  // tile-rows of the chunk, in images
    const int prof = prof_begin(s, PROF_WINO_INPUT, 0, 0,
                                4.0 * (imgs * g.C_in * g.H * g.W + static_cast<double>(tile) * tile * Tc * g.C_in));
    if (tile == 8) wino_input_kernel<8><<<grid, kXformThreads, 0, s>>>(in, V, g, R0, Tc, ncb);
    else wino_input_kernel<4><<<grid, kXformThreads, 0, s>>>(in, V, g, R0, Tc, ncb);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

template <bool CLIP>
static void wino_output_launch(int tile, dim3 grid, const float* M, float* out, const WinoGeom& g, int R0, int Tc,
                               const ConvEpilogue& e, int ncb, cudaStream_t s) {
    if (tile == 8) {
        if (e.pool) wino_output_kernel<8, true, CLIP><<<grid, kXformThreads, 0, s>>>(M, out, e.bias, g, R0, Tc, e.act, e.lo, e.hi, ncb);
        else wino_output_kernel<8, false, CLIP><<<grid, kXformThreads, 0, s>>>(M, out, e.bias, g, R0, Tc, e.act, e.lo, e.hi, ncb);
    } else {
        if (e.pool) wino_output_kernel<4, true, CLIP><<<grid, kXformThreads, 0, s>>>(M, out, e.bias, g, R0, Tc, e.act, e.lo, e.hi, ncb);
        else wino_output_kernel<4, false, CLIP><<<grid, kXformThreads, 0, s>>>(M, out, e.bias, g, R0, Tc, e.act, e.lo, e.hi, ncb);
    }
}

int wino_output_transform(int tile, const float* M, float* out, const WinoGeom& g, int R0, int R1, const ConvEpilogue& e,
                          cudaStream_t s) {
    const int segs = ceil_div(g.tilesX, kSegTiles);
    const int Tc = (R1 - R0) * g.tilesX;
    dim3 grid(static_cast<unsigned>(segs) * (R1 - R0), ceil_div(g.C_out, kChBlock));
    int ncb = 0;
    if (static_cast<unsigned long long>(grid.x) * grid.y < 0x7fffffffULL) {
        ncb = static_cast<int>(grid.y);
        grid = dim3(grid.x * grid.y, 1);
    }
    const double imgs = static_cast<double>(R1 - R0) / g.tilesY;  // tile-rows of the chunk, in images
    const double out_px = e.pool ? static_cast<double>((g.OH + 1) / 2) * ((g.OW + 1) / 2) : static_cast<double>(g.OH) * g.OW;
    const int prof = prof_begin(s, PROF_WINO_OUTPUT, 0, 0,
                                4.0 * (imgs * g.C_out * out_px + static_cast<double>(tile) * tile * Tc * g.C_out));
    if (e.act == 2) wino_output_launch<true>(tile, grid, M, out, g, R0, Tc, e, ncb, s);
    else wino_output_launch<false>(tile, grid, M, out, g, R0, Tc, e, ncb, s);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
