// Depthwise convolution (group == channels).
//
// Replaces DEPTHWISE_Forward (/root/reference/src/booster/avx/booster.cpp:136-160) -> dwConv_template /
// globalDwConv (avx/depthwise.cpp:161-207, 30-55) and the hand-unrolled NEON dwConvs1/dwConvs2
// (arm/depthwise.cpp:166,803).  The op is HBM-bound (18 FLOP per 8 bytes): the 3x3 kernels keep a 3-row
// sliding window in registers, read every input element once per warp with coalesced row loads and fetch
// the horizontal neighbours with warp shuffles (only the two edge lanes issue an extra halo load).
// Zero padding comes from the bounds checks — no padded copy (the reference's pad_input) is made.
// Stride semantics are the geometric ones; the reference swaps stride_w/stride_h in its index
// (depthwise.cpp:184), which is identical whenever stride_h == stride_w (all models in scope).
#include "depthwise.cuh"
#include "common.cuh"

#include <stdint.h>
#include <stdlib.h>

#include <algorithm>

namespace fcuda {

constexpr int kDwRows = 16;  // output rows marched by one warp

template <int STRIDE, bool CLIP>
__global__ void __launch_bounds__(128)
dw3x3_shuffle_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ out, int C, int H, int W, int OH, int OW, int act, float lo, float hi,
                     long long items, int xstrips, int ystrips) {
    const long long item = static_cast<long long>(blockIdx.x) * 4 + (threadIdx.x >> 5);
    if (item >= items) return;
    const int lane = threadIdx.x & 31;
    const int xs = static_cast<int>(item % xstrips);
    const long long t = item / xstrips;
    const int ys = static_cast<int>(t % ystrips);
    const long long plane = t / ystrips;  // n * C + c
    const int c = static_cast<int>(plane % C);
    const float* ip = in + plane * H * W;
    float* op = out + plane * OH * OW;

    float k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) k[i] = __ldg(w + c * 9 + i);
    const float bv = bias ? __ldg(bias + c) : 0.f;

    const int ox = xs * 32 + lane;
    const int oy0 = ys * kDwRows;
    const int oy1 = min(oy0 + kDwRows, OH);

    // The op is latency-bound unless many row loads are in flight per warp (measured: one row at a time = 29 % of HBM
    // bandwidth with 40 resident warps).  So input rows are fetched in batches — all global loads of a batch are issued
    // before the first shuffle (a shuffle waits for its load and would serialise the loads behind it) — and the
    // horizontal neighbours come from warp shuffles; only lanes 0 / 31 issue one extra (halo) load per row.
    auto fma3 = [&](float v, int kr, float l, float m, float r) {
        v = fmaf(k[kr * 3 + 0], l, v);
        v = fmaf(k[kr * 3 + 1], m, v);
        return fmaf(k[kr * 3 + 2], r, v);
    };
    if (STRIDE == 1) {
        constexpr int NB = 4;  // output rows per batch == new input rows per batch
        const int ix = ox;     // centre column (pad_left == 1)
        const int hx = lane == 0 ? ix - 1 : ix + 1;  // halo column of the edge lanes
        const bool m_ok = ix < W, h_ok = (lane == 0 || lane == 31) && hx >= 0 && hx < W;
        auto fetch = [&](int iy, float& m, float& h) {
            const bool row_ok = iy >= 0 && iy < H;
            const float* rp = ip + static_cast<long long>(iy) * W;
            m = (row_ok && m_ok) ? __ldg(rp + ix) : 0.f;
            h = (row_ok && h_ok) ? __ldg(rp + hx) : 0.f;
        };
        auto spread = [&](float m, float h, float& l, float& r) {
            l = __shfl_up_sync(0xffffffffu, m, 1);
            r = __shfl_down_sync(0xffffffffu, m, 1);
            if (lane == 0) l = h;
            if (lane == 31) r = h;
        };
        float am, ah, bm, bh, al, ar, bl, br;
        fetch(oy0 - 1, am, ah);
        fetch(oy0, bm, bh);
        spread(am, ah, al, ar);
        spread(bm, bh, bl, br);
        for (int oy = oy0; oy < oy1; oy += NB) {
            float cm[NB], ch[NB], cl[NB], cr[NB];
#pragma unroll
            for (int i = 0; i < NB; ++i) fetch(oy + 1 + i, cm[i], ch[i]);
#pragma unroll
            for (int i = 0; i < NB; ++i) spread(cm[i], ch[i], cl[i], cr[i]);
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                // window rows: (a, b, c0), (b, c0, c1), (c0, c1, c2), (c1, c2, c3)
                const float tl = i == 0 ? al : i == 1 ? bl : cl[i - 2], tm = i == 0 ? am : i == 1 ? bm : cm[i - 2],
                            tr = i == 0 ? ar : i == 1 ? br : cr[i - 2];
                const float ml = i == 0 ? bl : cl[i - 1], mm = i == 0 ? bm : cm[i - 1], mr = i == 0 ? br : cr[i - 1];
                float v = fma3(bv, 0, tl, tm, tr);
                v = fma3(v, 1, ml, mm, mr);
                v = fma3(v, 2, cl[i], cm[i], cr[i]);
                if (act) v = act_clamp<CLIP>(v, lo, hi);
                if (ox < OW && oy + i < oy1) op[static_cast<long long>(oy + i) * OW + ox] = v;
            }
            al = cl[NB - 2]; am = cm[NB - 2]; ar = cr[NB - 2];
            bl = cl[NB - 1]; bm = cm[NB - 1]; br = cr[NB - 1];
        }
    } else {
        constexpr int NB = 2;  // output rows per batch (4 new input rows)
        const int ix = 2 * ox;  // centre column 2*ox - 1 + 1
        const bool m_ok = ix < W, r_ok = ix + 1 < W, h_ok = lane == 0 && ix - 1 >= 0 && ix - 1 < W;
        auto fetch = [&](int iy, float& m, float& r, float& h) {
            const bool row_ok = iy >= 0 && iy < H;
            const float* rp = ip + static_cast<long long>(iy) * W;
            m = (row_ok && m_ok) ? __ldg(rp + ix) : 0.f;
            r = (row_ok && r_ok) ? __ldg(rp + ix + 1) : 0.f;
            h = (row_ok && h_ok) ? __ldg(rp + ix - 1) : 0.f;
        };
        auto spread = [&](float r, float h, float& l) {
            l = __shfl_up_sync(0xffffffffu, r, 1);
            if (lane == 0) l = h;
        };
        float am, ar, ah, al;
        fetch(2 * oy0 - 1, am, ar, ah);
        spread(ar, ah, al);
        for (int oy = oy0; oy < oy1; oy += NB) {
            float cm[2 * NB], cr[2 * NB], ch[2 * NB], cl[2 * NB];
#pragma unroll
            for (int i = 0; i < 2 * NB; ++i) fetch(2 * oy + i, cm[i], cr[i], ch[i]);
#pragma unroll
            for (int i = 0; i < 2 * NB; ++i) spread(cr[i], ch[i], cl[i]);
#pragma unroll
            for (int i = 0; i < NB; ++i) {
                // output row oy+i reads input rows 2(oy+i)-1, 2(oy+i), 2(oy+i)+1 = (a | c[2i-1]), c[2i], c[2i+1]
                const float tl = i == 0 ? al : cl[2 * i - 1], tm = i == 0 ? am : cm[2 * i - 1], tr = i == 0 ? ar : cr[2 * i - 1];
                float v = fma3(bv, 0, tl, tm, tr);
                v = fma3(v, 1, cl[2 * i], cm[2 * i], cr[2 * i]);
                v = fma3(v, 2, cl[2 * i + 1], cm[2 * i + 1], cr[2 * i + 1]);
                if (act) v = act_clamp<CLIP>(v, lo, hi);
                if (ox < OW && oy + i < oy1) op[static_cast<long long>(oy + i) * OW + ox] = v;
            }
            al = cl[2 * NB - 1]; am = cm[2 * NB - 1]; ar = cr[2 * NB - 1];
        }
    }
}

// Vectorised variant for wide planes (MobileNet's 112- and 56-wide stages): a lane owns VEC consecutive output columns, so a
// warp request is VEC x 128 bytes (the scalar kernel above keeps too few bytes in flight: 0.43 of HBM bandwidth, latency
// bound) and loads / stores / shuffles are amortised over VEC outputs; the inner loop is then the 9 FMAs per output.
//   stride 1: per input row a lane loads VEC floats at its first output column; left / right neighbours of the lane's span
//             come from the adjacent lanes by shuffle, the strip's outer halo by one extra load on lanes 0 / 31
//   stride 2: per input row a lane loads 2*VEC floats at column 2*ox0; the left halo (column 2*ox0 - 1) is the previous lane's
//             last element
// Requires pad 1, W % VEC == 0 (stride 1) or W % (2*VEC) == 0 (stride 2): vector accesses stay aligned and all-or-nothing.
template <int N> struct VecT;
template <> struct VecT<1> { typedef float type; };
template <> struct VecT<2> { typedef float2 type; };
template <> struct VecT<4> { typedef float4 type; };

template <int STRIDE, int VEC, bool CLIP>
__global__ void __launch_bounds__(128)
dw3x3_vec_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                 float* __restrict__ out, int C, int H, int W, int OH, int OW, int act, float lo, float hi, long long items,
                 int xstrips, int ystrips) {
    constexpr int LW = STRIDE * VEC;  // floats loaded per lane and input row
    typedef typename VecT<LW>::type LoadT;
    typedef typename VecT<VEC>::type StoreT;
    const long long item = static_cast<long long>(blockIdx.x) * 4 + (threadIdx.x >> 5);
    if (item >= items) return;
    const int lane = threadIdx.x & 31;
    const int xs = static_cast<int>(item % xstrips);
    const long long t = item / xstrips;
    const int ys = static_cast<int>(t % ystrips);
    const long long plane = t / ystrips;  // n * C + c
    const int c = static_cast<int>(plane % C);
    const float* ip = in + plane * H * W;
    float* op = out + plane * OH * OW;

    float k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) k[i] = __ldg(w + c * 9 + i);
    const float bv = bias ? __ldg(bias + c) : 0.f;

    const int ox0 = (xs * 32 + lane) * VEC;      // first output column of this lane
    const int ix0 = ox0 * STRIDE;                // first loaded input column (window of ox0 = ix0 - 1 .. ix0 + 1)
    const int oy0 = ys * kDwRows;
    const int oy1 = min(oy0 + kDwRows, OH);
    const bool in_ok = ix0 < W;                  // W % LW == 0: the whole span is inside or outside
    const bool lh_ok = lane == 0 && ix0 - 1 >= 0 && ix0 - 1 < W;                      // strip's left halo column
    const bool rh_ok = STRIDE == 1 && lane == 31 && ix0 + VEC < W;                    // strip's right halo (stride 1 only)

    struct Row { float m[LW]; float l, r; };
    auto fetch = [&](int iy, Row& row) {
        const bool row_ok = iy >= 0 && iy < H;
        const float* rp = ip + static_cast<long long>(iy) * W;
        if (row_ok && in_ok) {
            const LoadT v = __ldg(reinterpret_cast<const LoadT*>(rp + ix0));
            const float* f = reinterpret_cast<const float*>(&v);
#pragma unroll
            for (int j = 0; j < LW; ++j) row.m[j] = f[j];
        } else {
#pragma unroll
            for (int j = 0; j < LW; ++j) row.m[j] = 0.f;
        }
        row.l = (row_ok && lh_ok) ? __ldg(rp + ix0 - 1) : 0.f;
        row.r = (row_ok && rh_ok) ? __ldg(rp + ix0 + VEC) : 0.f;
    };
    auto spread = [&](Row& row) {  // after ALL loads of a batch were issued (a shuffle waits for its load)
        const float l = __shfl_up_sync(0xffffffffu, row.m[LW - 1], 1);
        if (lane != 0) row.l = l;
        if (STRIDE == 1) {
            const float r = __shfl_down_sync(0xffffffffu, row.m[0], 1);
            if (lane != 31) row.r = r;
        }
    };
    // horizontal 3-tap of kernel row kr for output j: inputs at columns STRIDE*j - 1, STRIDE*j, STRIDE*j + 1 of the span
    auto tap = [&](float v, int kr, const Row& row, int j) {
        const int cidx = STRIDE * j;
        const float a = cidx == 0 ? row.l : row.m[cidx - 1];
        const float b = row.m[cidx];
        const float d = cidx + 1 < LW ? row.m[cidx + 1] : row.r;
        v = fmaf(k[kr * 3 + 0], a, v);
        v = fmaf(k[kr * 3 + 1], b, v);
        return fmaf(k[kr * 3 + 2], d, v);
    };
    auto emit = [&](int oy, const Row& r0, const Row& r1, const Row& r2) {
        __align__(16) float o[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            float v = tap(bv, 0, r0, j);
            v = tap(v, 1, r1, j);
            v = tap(v, 2, r2, j);
            o[j] = act ? act_clamp<CLIP>(v, lo, hi) : v;
        }
        if (ox0 < OW && oy < oy1) *reinterpret_cast<StoreT*>(op + static_cast<long long>(oy) * OW + ox0) = *reinterpret_cast<StoreT*>(o);
    };

    if (STRIDE == 1) {
        constexpr int NB = 4;
        Row a, b;
        fetch(oy0 - 1, a);
        fetch(oy0, b);
        spread(a);
        spread(b);
        for (int oy = oy0; oy < oy1; oy += NB) {
            Row cr[NB];
#pragma unroll
            for (int i = 0; i < NB; ++i) fetch(oy + 1 + i, cr[i]);
#pragma unroll
            for (int i = 0; i < NB; ++i) spread(cr[i]);
            emit(oy, a, b, cr[0]);
            emit(oy + 1, b, cr[0], cr[1]);
            emit(oy + 2, cr[0], cr[1], cr[2]);
            emit(oy + 3, cr[1], cr[2], cr[3]);
            a = cr[NB - 2];
            b = cr[NB - 1];
        }
    } else {
        constexpr int NB = 2;  // output rows per batch (4 new input rows)
        Row a;
        fetch(2 * oy0 - 1, a);
        spread(a);
        for (int oy = oy0; oy < oy1; oy += NB) {
            Row cr[2 * NB];
#pragma unroll
            for (int i = 0; i < 2 * NB; ++i) fetch(2 * oy + i, cr[i]);
#pragma unroll
            for (int i = 0; i < 2 * NB; ++i) spread(cr[i]);
            emit(oy, a, cr[0], cr[1]);
            emit(oy + 1, cr[1], cr[2], cr[3]);
            a = cr[2 * NB - 1];
        }
    }
}

// 3x3 depthwise on small planes (MobileNet's 14x14 and 7x7 stages, where a 32-wide strip would idle most lanes): one warp
// per (image, channel) plane.  The plane goes to shared memory with a zero halo of one pixel, then every lane computes
// output pixels lane, lane+32, ...; row/column come from a 16-bit reciprocal multiply (exact for planes <= 34x34).
template <int STRIDE, bool CLIP>
__global__ void __launch_bounds__(128)
dw3x3_plane_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                   float* __restrict__ out, int C, int H, int W, int OH, int OW, int pad_top, int pad_left,
                   int act, float lo, float hi, long long planes) {
    extern __shared__ float dw_smem[];
    const int PW = W + 2, PH = H + 2;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long plane = static_cast<long long>(blockIdx.x) * 4 + warp;
    if (plane >= planes) return;
    float* tile = dw_smem + warp * PH * PW;
    const int c = static_cast<int>(plane % C);
    const float* ip = in + plane * H * W;
    const unsigned rcp_pw = (65536u + PW - 1) / PW, rcp_ow = (65536u + OW - 1) / OW;
    // eight loads in flight per lane, then the eight shared-memory stores (a store right behind its load would make the
    // next load wait for it)
    const unsigned n_tile = static_cast<unsigned>(PH * PW);
    for (unsigned base = 0; base < n_tile; base += 256) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const unsigned i = base + j * 32 + lane;
            const unsigned y = (i * rcp_pw) >> 16, x = i - y * PW;
            const int iy = static_cast<int>(y) - 1, ix = static_cast<int>(x) - 1;
            v[j] = (i < n_tile && iy >= 0 && iy < H && ix >= 0 && ix < W) ? __ldg(ip + iy * W + ix) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const unsigned i = base + j * 32 + lane;
            if (i < n_tile) tile[i] = v[j];
        }
    }
    float k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) k[i] = __ldg(w + c * 9 + i);
    const float bv = bias ? __ldg(bias + c) : 0.f;
    __syncwarp();
    float* op = out + plane * OH * OW;
    for (unsigned o = lane; o < static_cast<unsigned>(OH * OW); o += 32) {
        const unsigned oy = (o * rcp_ow) >> 16, ox = o - oy * OW;
        // window start in image coordinates is (oy*S - pad_top, ox*S - pad_left); +1 for the halo
        const float* t = tile + (oy * STRIDE + 1 - pad_top) * PW + (ox * STRIDE + 1 - pad_left);
        float v = bv;
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
            for (int x = 0; x < 3; ++x) v = fmaf(k[u * 3 + x], t[u * PW + x], v);
        if (act) v = act_clamp<CLIP>(v, lo, hi);
        op[o] = v;
    }
}

// 3x3 / stride 1 / pad 1 on planes up to 16 x 16 (MobileNet's five 14x14 layers and the 7x7 one): a lane owns ONE COLUMN of
// one plane — LP = 16 or 8 lanes per plane, 2 or 4 planes per warp — loads that column's H values up front (H independent
// loads in flight per lane), gets the left / right neighbours of every row with sub-warp shuffles and writes its output
// column.  ~13 instructions per output row and lane; the shared-memory plane kernel above needs ~300 warp instructions per
// 14x14 plane and is issue-bound there.
template <int LP, bool CLIP>
__global__ void __launch_bounds__(128)
dw3x3_cols_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                  float* __restrict__ out, int C, int H, int W, int act, float lo, float hi, long long planes) {
    constexpr int PPW = 32 / LP;  // planes per warp
    const int lane = threadIdx.x & 31, sub = lane / LP, col = lane % LP;
    const long long plane = (static_cast<long long>(blockIdx.x) * 4 + (threadIdx.x >> 5)) * PPW + sub;
    const bool p_ok = plane < planes, ok = p_ok && col < W;
    const long long pl = p_ok ? plane : 0;
    const int c = static_cast<int>(pl % C);
    const float* ip = in + pl * H * W + col;
    float k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) k[i] = __ldg(w + c * 9 + i);
    const float bv = bias ? __ldg(bias + c) : 0.f;
    float m[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) m[r] = (ok && r < H) ? __ldg(ip + r * W) : 0.f;
    float l[16], rr[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) {  // lanes with col >= W hold zeros, so the right edge needs no special case
        const float a = __shfl_up_sync(0xffffffffu, m[r], 1, LP);
        const float b = __shfl_down_sync(0xffffffffu, m[r], 1, LP);
        l[r] = col == 0 ? 0.f : a;
        rr[r] = col == LP - 1 ? 0.f : b;
    }
    float* op = out + pl * H * W + col;
#pragma unroll
    for (int oy = 0; oy < 16; ++oy) {
        if (oy < H) {
            float v = bv;
            if (oy > 0) { v = fmaf(k[0], l[oy - 1], v); v = fmaf(k[1], m[oy - 1], v); v = fmaf(k[2], rr[oy - 1], v); }
            v = fmaf(k[3], l[oy], v); v = fmaf(k[4], m[oy], v); v = fmaf(k[5], rr[oy], v);
            if (oy + 1 < 16) { v = fmaf(k[6], l[oy + 1], v); v = fmaf(k[7], m[oy + 1], v); v = fmaf(k[8], rr[oy + 1], v); }
            if (act) v = act_clamp<CLIP>(v, lo, hi);
            if (ok) op[oy * W] = v;
        }
    }
}

// Dilated 3x3 / stride 1 depthwise (DeepLab's atrous backbones: pad = dilation on 33x33 or 65x65 planes, dilations 2 to 18).
// One CTA per strip of up to kDilRows output rows of one plane.  The CTA stages the strip's input box, (rows + 2 dh) x
// (OW + 2 dw), in shared memory with zeros where the box leaves the image, so the compute loop has no bounds checks.  The
// image rows of the box are one contiguous span of the input: it is read with 16-byte loads between a scalar head and tail
// whatever the plane width or pointer alignment, and each element is scattered to its box row by a reciprocal multiply.
// Each input element comes from HBM once per layer; the 2 dh halo rows shared by neighbouring strips come again from L2.
// A thread then marches one chain of outputs dh rows apart (rows rho, rho + dh, ...): consecutive outputs of a chain share
// two of their three window rows, so each step reads one new window row (3 VEC values) from shared memory.  VEC = 4: a
// thread owns four consecutive columns and stores them as one float4 (OW % 4 == 0 and a 16-byte aligned output).
constexpr int kDilThreads = 128;
constexpr int kDilRows = 64;       // output rows per strip, before balancing the strips of a plane
constexpr int kDilChain = 4;       // outputs per chain segment: one thread's work item
constexpr int kDilMaxBox = 12288;  // floats of the staged box (48 KB: no dynamic shared-memory opt-in)

template <int VEC, bool CLIP>
__global__ void __launch_bounds__(kDilThreads)
dw3x3_dilated_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ out, DwGeom g, int TH, int strips, int BW, unsigned w_rcp, int act, float lo,
                     float hi) {
    extern __shared__ float box[];
    const int tid = threadIdx.x;
    const long long plane = blockIdx.x / strips;  // n * C + c
    const int strip = static_cast<int>(blockIdx.x - plane * strips);
    const int c = static_cast<int>(plane % g.C);
    const int dh = g.dil_h, dw = g.dil_w;
    const int oy0 = strip * TH, th = min(TH, g.OH - oy0);
    const int BH = th + 2 * dh;
    const int by0 = oy0 - g.pad_top;  // image row of box row 0
    // box rows [r_lo, r_hi) hold image rows; the others, and the pad columns of these, are zero
    const int r_lo = min(max(0, -by0), BH), r_hi = max(r_lo, min(BH, g.H - by0));
    for (int i = tid; i < r_lo * BW; i += kDilThreads) box[i] = 0.f;
    for (int i = r_hi * BW + tid; i < BH * BW; i += kDilThreads) box[i] = 0.f;
    const int padl = min(g.pad_left, BW), padr = max(0, BW - g.pad_left - g.W), pc = padl + padr;
    for (int i = tid; i < (r_hi - r_lo) * pc; i += kDilThreads) {
        const int r = r_lo + i / pc, x = i % pc;
        box[r * BW + (x < padl ? x : g.pad_left + g.W + x - padl)] = 0.f;
    }
    const float* src = in + plane * g.H * g.W + static_cast<long long>(by0 + r_lo) * g.W;
    const int n = (r_hi - r_lo) * g.W;
    // e < n <= kDilMaxBox keeps e * W far below 2^32: __umulhi(e, ceil(2^32 / W)) is exactly e / W
    auto put = [&](int e, float v) {
        const int r = static_cast<int>(__umulhi(static_cast<unsigned>(e), w_rcp));
        const int col = g.pad_left + e - r * g.W;
        if (col < BW) box[(r_lo + r) * BW + col] = v;
    };
    const int head = min(n, static_cast<int>(((16u - (static_cast<unsigned>(reinterpret_cast<uintptr_t>(src)) & 15u)) & 15u) >> 2));
    if (tid < head) put(tid, __ldg(src + tid));
    const int nq = (n - head) >> 2;
    const float4* s4 = reinterpret_cast<const float4*>(src + head);
    for (int q0 = tid; q0 < nq; q0 += 4 * kDilThreads) {
        float4 v[4];  // four 16-byte loads in flight before the first shared-memory store
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int q = q0 + j * kDilThreads;
            v[j] = q < nq ? __ldg(s4 + q) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int q = q0 + j * kDilThreads;
            if (q < nq) {
                const int e = head + 4 * q;
                put(e, v[j].x); put(e + 1, v[j].y); put(e + 2, v[j].z); put(e + 3, v[j].w);
            }
        }
    }
    const int tail = head + 4 * nq + tid;
    if (tail < n) put(tail, __ldg(src + tail));
    float k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) k[i] = __ldg(w + c * 9 + i);
    const float bv = bias ? __ldg(bias + c) : 0.f;
    __syncthreads();

    const int chains = min(dh, th), segs = ((th + dh - 1) / dh + kDilChain - 1) / kDilChain, xq = g.OW / VEC;
    float* op = out + plane * g.OH * g.OW + static_cast<long long>(oy0) * g.OW;
    for (int it = tid; it < xq * chains * segs; it += kDilThreads) {
        const int ox = (it % xq) * VEC, rest = it / xq, rho = rest % chains, m0 = rest / chains * kDilChain;
        const int len = (th - rho + dh - 1) / dh;  // outputs of chain rho
        if (m0 >= len) continue;
        const int m1 = min(m0 + kDilChain, len);
        float a[3][VEC], b[3][VEC], cur[3][VEC];
        auto row = [&](int m, float (&v)[3][VEC]) {  // box row rho + m * dh, columns ox + j * dw + i
            const float* p = box + (rho + m * dh) * BW + ox;
#pragma unroll
            for (int j = 0; j < 3; ++j)
#pragma unroll
                for (int i = 0; i < VEC; ++i) v[j][i] = p[j * dw + i];
        };
        row(m0, a);
        row(m0 + 1, b);
        for (int m = m0; m < m1; ++m) {
            row(m + 2, cur);
            __align__(16) float o[VEC];
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                float v = bv;
#pragma unroll
                for (int j = 0; j < 3; ++j) v = fmaf(k[j], a[j][i], v);
#pragma unroll
                for (int j = 0; j < 3; ++j) v = fmaf(k[3 + j], b[j][i], v);
#pragma unroll
                for (int j = 0; j < 3; ++j) v = fmaf(k[6 + j], cur[j][i], v);
                o[i] = act ? act_clamp<CLIP>(v, lo, hi) : v;
            }
            float* dst = op + static_cast<long long>(rho + m * dh) * g.OW + ox;
            if (VEC == 4) *reinterpret_cast<float4*>(dst) = *reinterpret_cast<const float4*>(o);
            else dst[0] = o[0];
#pragma unroll
            for (int j = 0; j < 3; ++j)
#pragma unroll
                for (int i = 0; i < VEC; ++i) { a[j][i] = b[j][i]; b[j][i] = cur[j][i]; }
        }
    }
}

// Generic k x k / any stride / any padding / any dilation depthwise: one thread per output element.
template <bool CLIP>
__global__ void __launch_bounds__(256)
dw_generic_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                  float* __restrict__ out, DwGeom g, int act, float lo, float hi, long long total) {
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int ox = static_cast<int>(idx % g.OW);
    long long t = idx / g.OW;
    const int oy = static_cast<int>(t % g.OH);
    const long long plane = t / g.OH;
    const int c = static_cast<int>(plane % g.C);
    const float* ip = in + plane * g.H * g.W;
    const float* kp = w + static_cast<size_t>(c) * g.KH * g.KW;
    float v = 0.f;
    for (int u = 0; u < g.KH; ++u) {
        const int iy = oy * g.stride_h - g.pad_top + u * g.dil_h;
        if (iy < 0 || iy >= g.H) continue;
        for (int x = 0; x < g.KW; ++x) {
            const int ix = ox * g.stride_w - g.pad_left + x * g.dil_w;
            if (ix < 0 || ix >= g.W) continue;
            v = fmaf(__ldg(ip + static_cast<long long>(iy) * g.W + ix), __ldg(kp + u * g.KW + x), v);
        }
    }
    if (bias) v += __ldg(bias + c);
    if (act) v = act_clamp<CLIP>(v, lo, hi);
    out[idx] = v;
}

template <bool CLIP>
static void dw_generic_launch(const float* in, const float* w, float* out, const DwGeom& g, const ConvEpilogue& e, int batch,
                              cudaStream_t s) {
    const long long total = static_cast<long long>(batch) * g.C * g.OH * g.OW;
    dw_generic_kernel<CLIP><<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(in, w, e.bias, out, g, e.act, e.lo, e.hi, total);
}

// Strip height and box width of dw3x3_dilated_kernel for a dilated layer; false when the layer is not 3x3 / stride 1 or a
// strip of one output row would not fit the box.
static bool dil_strips(const DwGeom& g, int* TH, int* strips, int* BW) {
    if (g.KH != 3 || g.KW != 3 || g.stride_h != 1 || g.stride_w != 1 || g.W < 2) return false;
    const int bw = g.OW + 2 * g.dil_w;
    const int fit = kDilMaxBox / bw - 2 * g.dil_h;  // most output rows whose box fits
    if (fit < 1) return false;
    const int n = ceil_div(g.OH, std::min(kDilRows, fit));
    *strips = n;
    *TH = ceil_div(g.OH, n);  // balanced strips
    *BW = bw;
    return true;
}

// The kernel choice of depthwise_forward; CLIP selects the Clip instantiations (act == 2).
template <bool CLIP>
static void dw_launch(const float* in, const float* w, float* out, const DwGeom& g, const ConvEpilogue& e, int batch,
                      cudaStream_t s) {
    if (g.dil_h > 1 || g.dil_w > 1) {
        int TH, strips, BW;
        if (!dil_strips(g, &TH, &strips, &BW)) return dw_generic_launch<CLIP>(in, w, out, g, e, batch, s);
        const unsigned blocks = static_cast<unsigned>(static_cast<long long>(batch) * g.C * strips);
        const int smem = (TH + 2 * g.dil_h) * BW * static_cast<int>(sizeof(float));
        const unsigned w_rcp = static_cast<unsigned>(((1ull << 32) + g.W - 1) / g.W);
        if (g.OW % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0)
            dw3x3_dilated_kernel<4, CLIP><<<blocks, kDilThreads, smem, s>>>(in, w, e.bias, out, g, TH, strips, BW, w_rcp, e.act,
                                                                          e.lo, e.hi);
        else
            dw3x3_dilated_kernel<1, CLIP><<<blocks, kDilThreads, smem, s>>>(in, w, e.bias, out, g, TH, strips, BW, w_rcp, e.act,
                                                                          e.lo, e.hi);
        return;
    }
    const bool k3 = g.KH == 3 && g.KW == 3 && g.pad_top == 1 && g.pad_left == 1 && g.stride_h == g.stride_w &&
                    (g.stride_h == 1 || g.stride_h == 2) && g.OW >= 24;
    // vector width: the widest VEC whose strips (32 * VEC outputs) still fill most lanes and keep accesses aligned
    const bool vec_off = tune_get(TUNE_DW_VEC) == 0;
    const uintptr_t ia = reinterpret_cast<uintptr_t>(in), oa = reinterpret_cast<uintptr_t>(out);
    int vec = 1;
    if (k3 && !vec_off && g.stride_h == 1 && g.OW == g.W) {
        // float4 / float2 loads and stores: in and out aligned to the access width (a C ABI caller may pass any float*)
        if (g.W % 4 == 0 && g.OW >= 96 && ((ia | oa) & 15) == 0) vec = 4;
        else if (g.W % 2 == 0 && g.OW >= 48 && ((ia | oa) & 7) == 0) vec = 2;
    } else if (k3 && !vec_off && g.stride_h == 2 && g.W == 2 * g.OW) {
        // float4 loads, float2 stores: in 16-byte, out 8-byte aligned
        if (g.W % 4 == 0 && g.OW >= 48 && (ia & 15) == 0 && (oa & 7) == 0) vec = 2;
    }
    if (k3 && vec > 1) {
        const int xstrips = ceil_div(g.OW, 32 * vec), ystrips = ceil_div(g.OH, kDwRows);
        const long long items = static_cast<long long>(batch) * g.C * xstrips * ystrips;
        const unsigned blocks = static_cast<unsigned>((items + 3) / 4);
#define DW_VEC_LAUNCH(S, V) dw3x3_vec_kernel<S, V, CLIP><<<blocks, 128, 0, s>>>(in, w, e.bias, out, g.C, g.H, g.W, g.OH, g.OW, e.act, e.lo, e.hi, items, xstrips, ystrips)
        if (g.stride_h == 1 && vec == 4) DW_VEC_LAUNCH(1, 4);
        else if (g.stride_h == 1) DW_VEC_LAUNCH(1, 2);
        else DW_VEC_LAUNCH(2, 2);
#undef DW_VEC_LAUNCH
    } else if (k3) {
        const int xstrips = ceil_div(g.OW, 32), ystrips = ceil_div(g.OH, kDwRows);
        const long long items = static_cast<long long>(batch) * g.C * xstrips * ystrips;
        const unsigned blocks = static_cast<unsigned>((items + 3) / 4);
        if (g.stride_h == 1)
            dw3x3_shuffle_kernel<1, CLIP><<<blocks, 128, 0, s>>>(in, w, e.bias, out, g.C, g.H, g.W, g.OH, g.OW, e.act, e.lo, e.hi, items,
                                                            xstrips, ystrips);
        else
            dw3x3_shuffle_kernel<2, CLIP><<<blocks, 128, 0, s>>>(in, w, e.bias, out, g.C, g.H, g.W, g.OH, g.OW, e.act, e.lo, e.hi, items,
                                                            xstrips, ystrips);
    } else if (!vec_off && g.KH == 3 && g.KW == 3 && g.pad_top == 1 && g.pad_left == 1 && g.stride_h == 1 && g.stride_w == 1 &&
               g.H <= 16 && g.W <= 16 && g.OH == g.H && g.OW == g.W) {
        const long long planes_ll = static_cast<long long>(batch) * g.C;
        if (g.W <= 8) {
            const unsigned blocks = static_cast<unsigned>((planes_ll + 15) / 16);
            dw3x3_cols_kernel<8, CLIP><<<blocks, 128, 0, s>>>(in, w, e.bias, out, g.C, g.H, g.W, e.act, e.lo, e.hi, planes_ll);
        } else {
            const unsigned blocks = static_cast<unsigned>((planes_ll + 7) / 8);
            dw3x3_cols_kernel<16, CLIP><<<blocks, 128, 0, s>>>(in, w, e.bias, out, g.C, g.H, g.W, e.act, e.lo, e.hi, planes_ll);
        }
    } else if (g.KH == 3 && g.KW == 3 && (g.pad_top == 0 || g.pad_top == 1) && (g.pad_left == 0 || g.pad_left == 1) &&
               g.stride_h == g.stride_w && (g.stride_h == 1 || g.stride_h == 2) && g.H <= 34 && g.W <= 34 &&
               (g.OH - 1) * g.stride_h - g.pad_top + 2 <= g.H && (g.OW - 1) * g.stride_w - g.pad_left + 2 <= g.W) {
        // (the last window may reach one pixel past the image: that is the zero halo)
        const long long planes_ll = static_cast<long long>(batch) * g.C;
        const unsigned blocks = static_cast<unsigned>((planes_ll + 3) / 4);
        const int smem = 4 * (g.H + 2) * (g.W + 2) * static_cast<int>(sizeof(float));
        if (g.stride_h == 1)
            dw3x3_plane_kernel<1, CLIP><<<blocks, 128, smem, s>>>(in, w, e.bias, out, g.C, g.H, g.W, g.OH, g.OW, g.pad_top,
                                                             g.pad_left, e.act, e.lo, e.hi, planes_ll);
        else
            dw3x3_plane_kernel<2, CLIP><<<blocks, 128, smem, s>>>(in, w, e.bias, out, g.C, g.H, g.W, g.OH, g.OW, g.pad_top,
                                                             g.pad_left, e.act, e.lo, e.hi, planes_ll);
    } else {
        dw_generic_launch<CLIP>(in, w, out, g, e, batch, s);
    }
}

int depthwise_forward(const float* in, const float* w, float* out, const DwGeom& geom, const ConvEpilogue& e, int batch,
                      cudaStream_t s) {
    DwGeom g = geom;
    g.dil_h = std::max(g.dil_h, 1);
    g.dil_w = std::max(g.dil_w, 1);
    const double planes = static_cast<double>(batch) * g.C;
    const int prof = prof_begin(s, PROF_DEPTHWISE, 2.0 * planes * g.OH * g.OW * g.KH * g.KW, 0,
                                4.0 * planes * (static_cast<double>(g.H) * g.W + static_cast<double>(g.OH) * g.OW));
    if (e.act == 2) dw_launch<true>(in, w, out, g, e, batch, s);
    else dw_launch<false>(in, w, out, g, e, batch, s);
    prof_end(prof, s);
    FCUDA_CHECK_LAUNCH();
    count_launch();
    return 0;
}

}  // namespace fcuda
