// SSD detection head: ncnn's Permute, a softmax over one axis, Caffe / ncnn PriorBox, and DetectionOutput (centre-size
// decode, per-class top-k and greedy NMS, merge over the classes) as stream-ordered kernels that allocate nothing, so a
// detection net stays on the device and inside one CUDA graph from pixels to boxes.
//
// DetectionOutput runs three kernels:
//   decode     one thread per (image, prior): the boxes into the workspace;
//   nms_class  one CTA per (image, class): radix-select the nms_top_k best candidates (score, then prior index), sort
//              them bitonically in shared memory, then sweep them in order; each box still standing suppresses the later
//              ones in parallel.  The kept keys go to the workspace in sorted order;
//   merge      one CTA per image: the same select and sort over the kept lists of all classes, then the output rows.
// Keys are 64 bits: an order-preserving image of the fp32 score above 32 bits of (0xffffffff - index), so one descending
// sort gives score descending and index ascending.
#include "activation.cuh"
#include "common.cuh"
#include "detection.cuh"

#include <float.h>
#include <math.h>
#include <stdint.h>

namespace fcuda {

namespace {

constexpr int kDetThreads = 512;
constexpr int kDetWarps = kDetThreads / 32;
constexpr int kMaxTopK = 1024;  // nms_top_k and keep_top_k limit: the candidates of one CTA live in shared memory
constexpr int kProposalMaxTopK = 8192;  // pre_nms_topN / after_nms_topN limit: 64 KB of keys in dynamic shared memory

// ---- Permute --------------------------------------------------------------------------------------------------------
// Input axis (0 = c, 1 = h, 2 = w) of each output axis, per ncnn order_type.
__constant__ int kPermAxes[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};

__global__ void __launch_bounds__(256)
permute_kernel(const float* __restrict__ in, float* __restrict__ out, int c, int h, int w, int order, long long total) {
    const int dims[3] = {c, h, w};
    const long long strides[3] = {static_cast<long long>(h) * w, w, 1};
    const int a0 = kPermAxes[order][0], a1 = kPermAxes[order][1], a2 = kPermAxes[order][2];
    const int d1 = dims[a1], d2 = dims[a2];
    const long long s0 = strides[a0], s1 = strides[a1], s2 = strides[a2];
    const long long image = static_cast<long long>(c) * h * w;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long n = idx / image;
        long long r = idx - n * image;
        const long long o2 = r % d2;
        r /= d2;
        const long long o1 = r % d1, o0 = r / d1;
        out[idx] = __ldg(in + n * image + o0 * s0 + o1 * s1 + o2 * s2);
    }
}

// Order 3, (c, h, w) -> (h, w, c): a transpose of the (c, h*w) matrix of each image through a 32 x 33 shared tile, so
// both the reads (along h*w) and the writes (along c) are coalesced.
constexpr int kTile = 32;
__global__ void __launch_bounds__(kTile * 8)
transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
    __shared__ float tile[kTile][kTile + 1];
    const size_t image = static_cast<size_t>(rows) * cols;
    const float* ip = in + image * blockIdx.z;
    float* op = out + image * blockIdx.z;
    const int c0 = blockIdx.x * kTile, r0 = blockIdx.y * kTile;
    for (int y = threadIdx.y; y < kTile; y += 8) {
        const int r = r0 + y, cc = c0 + threadIdx.x;
        if (r < rows && cc < cols) tile[y][threadIdx.x] = __ldg(ip + static_cast<size_t>(r) * cols + cc);
    }
    __syncthreads();
    for (int y = threadIdx.y; y < kTile; y += 8) {
        const int cc = c0 + y, r = r0 + threadIdx.x;
        if (r < rows && cc < cols) op[static_cast<size_t>(cc) * rows + r] = tile[threadIdx.x][y];
    }
}

// ---- softmax over one axis ------------------------------------------------------------------------------------------
// inner == 1: one warp per row of `len` contiguous values.
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ in, float* __restrict__ out, long long rows, int len) {
    const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float* ip = in + row * len;
    float* op = out + row * len;
    float m = -INFINITY;
    for (int j = lane; j < len; j += 32) m = fmaxf(m, ip[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < len; j += 32) {
        const float e = expf(ip[j] - m);
        op[j] = e;
        s += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int j = lane; j < len; j += 32) op[j] = op[j] / s;
}

// inner > 1: one thread per (image, outer, inner) column of `len` values `inner` apart; neighbouring threads read
// neighbouring columns.
__global__ void __launch_bounds__(256)
softmax_cols_kernel(const float* __restrict__ in, float* __restrict__ out, long long cols, int len, int inner) {
    const long long col = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= cols) return;
    const long long o = col / inner, i = col - o * inner;
    const size_t base = static_cast<size_t>(o) * len * inner + i;
    float m = -INFINITY;
    for (int j = 0; j < len; ++j) m = fmaxf(m, in[base + static_cast<size_t>(j) * inner]);
    float s = 0.f;
    for (int j = 0; j < len; ++j) {
        const float e = expf(in[base + static_cast<size_t>(j) * inner] - m);
        out[base + static_cast<size_t>(j) * inner] = e;
        s += e;
    }
    for (int j = 0; j < len; ++j) out[base + static_cast<size_t>(j) * inner] /= s;
}

// ---- PriorBox -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void put_box(float* o, float cx, float cy, float bw, float bh, float iw, float ih, int clip) {
    float v[4] = {__fdiv_rn(__fsub_rn(cx, __fmul_rn(bw, 0.5f)), iw), __fdiv_rn(__fsub_rn(cy, __fmul_rn(bh, 0.5f)), ih),
                  __fdiv_rn(__fadd_rn(cx, __fmul_rn(bw, 0.5f)), iw), __fdiv_rn(__fadd_rn(cy, __fmul_rn(bh, 0.5f)), ih)};
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = clip ? fminf(fmaxf(v[k], 0.f), 1.f) : v[k];
}

// one thread per feature-map location; out row 0 = boxes, row 1 (at 4 * total) = variances
__global__ void __launch_bounds__(256)
priorbox_kernel(float* __restrict__ out, const FcudaPriorBoxParam p, int per_loc, int fw, int fh, float iw, float ih,
                float step_w, float step_h) {
    const int loc = blockIdx.x * blockDim.x + threadIdx.x;
    if (loc >= fw * fh) return;
    const int y = loc / fw, x = loc - y * fw;
    const float cx = __fmul_rn(__fadd_rn(static_cast<float>(x), p.offset), step_w);
    const float cy = __fmul_rn(__fadd_rn(static_cast<float>(y), p.offset), step_h);
    const size_t total4 = static_cast<size_t>(fw) * fh * per_loc * 4;
    float* o = out + static_cast<size_t>(loc) * per_loc * 4;
    for (int k = 0; k < p.num_min_sizes; ++k) {
        const float mn = p.min_sizes[k];
        put_box(o, cx, cy, mn, mn, iw, ih, p.clip);
        o += 4;
        if (p.num_max_sizes > 0) {
            const float sz = sqrtf(__fmul_rn(mn, p.max_sizes[k]));
            put_box(o, cx, cy, sz, sz, iw, ih, p.clip);
            o += 4;
        }
        for (int a = 0; a < p.num_aspect_ratios; ++a) {
            const float ar = p.aspect_ratios[a];
            if (fabsf(ar - 1.f) < 1e-6f) continue;
            const float r = sqrtf(ar);
            put_box(o, cx, cy, __fmul_rn(mn, r), __fdiv_rn(mn, r), iw, ih, p.clip);
            o += 4;
            if (p.flip) {
                put_box(o, cx, cy, __fdiv_rn(mn, r), __fmul_rn(mn, r), iw, ih, p.clip);
                o += 4;
            }
        }
    }
    float* v = out + total4 + static_cast<size_t>(loc) * per_loc * 4;
    for (int j = 0; j < per_loc * 4; ++j) v[j] = p.variances[j & 3];
}

// ---- DetectionOutput ------------------------------------------------------------------------------------------------
// cx = var0 * l0 * pw + pcx, w = expf(var2 * l2) * pw, ...; every product and sum rounded on its own (no FMA)
__global__ void __launch_bounds__(256)
decode_kernel(float* __restrict__ boxes, const float* __restrict__ loc, const float* __restrict__ priors, int P,
              long long total) {
    const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int p = static_cast<int>(t % P);
    const float* pb = priors + static_cast<size_t>(p) * 4;
    const float* var = priors + static_cast<size_t>(P) * 4 + static_cast<size_t>(p) * 4;
    const float* l = loc + static_cast<size_t>(t) * 4;
    const float pw = __fsub_rn(pb[2], pb[0]), ph = __fsub_rn(pb[3], pb[1]);
    const float pcx = __fmul_rn(__fadd_rn(pb[0], pb[2]), 0.5f), pcy = __fmul_rn(__fadd_rn(pb[1], pb[3]), 0.5f);
    const float cx = __fadd_rn(__fmul_rn(__fmul_rn(var[0], l[0]), pw), pcx);
    const float cy = __fadd_rn(__fmul_rn(__fmul_rn(var[1], l[1]), ph), pcy);
    const float w = __fmul_rn(expf(__fmul_rn(var[2], l[2])), pw);
    const float h = __fmul_rn(expf(__fmul_rn(var[3], l[3])), ph);
    float* b = boxes + static_cast<size_t>(t) * 4;
    b[0] = __fsub_rn(cx, __fmul_rn(w, 0.5f));
    b[1] = __fsub_rn(cy, __fmul_rn(h, 0.5f));
    b[2] = __fadd_rn(cx, __fmul_rn(w, 0.5f));
    b[3] = __fadd_rn(cy, __fmul_rn(h, 0.5f));
}

// -0 takes the image of +0: the two are equal scores, ordered by class and prior like any other tie.  So the image does
// not give back the score's bits; the output row reads the score from conf.
__device__ __forceinline__ uint32_t orderable(float f) {
    uint32_t b = __float_as_uint(f);
    if (b == 0x80000000u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ unsigned long long make_key(uint32_t u, int i) {
    return (static_cast<unsigned long long>(u) << 32) | (0xffffffffu - static_cast<uint32_t>(i));
}
__device__ __forceinline__ int key_index(unsigned long long k) {
    return static_cast<int>(0xffffffffu - static_cast<uint32_t>(k));
}

// The scratch of select_top_k; the keys live apart, so their capacity is the caller's: SSD's and YOLO's CTAs hold
// kMaxTopK of them in SelectSmem, Proposal's up to kProposalMaxTopK in dynamic shared memory.
struct SelectScratch {
    int hist[256];
    int warp_sums[kDetWarps];
    int bcast[2];
};
struct SelectSmem {
    unsigned long long keys[kMaxTopK];
    SelectScratch s;
};

// Exclusive prefix of a 0/1 flag over the CTA in thread order; *total gets the CTA's sum.  Every thread calls it.
__device__ __forceinline__ int block_scan(int flag, int* total, SelectScratch& sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) sm.warp_sums[warp] = __popc(m);
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < kDetWarps; ++w) {
        const int c = sm.warp_sums[w];
        before += w < warp ? c : 0;
        sum += c;
    }
    __syncthreads();
    *total = sum;
    return before + __popc(m & ((1u << lane) - 1u));
}

__device__ __forceinline__ int block_sum(int v, SelectScratch& sm) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) sm.bcast[0] = 0;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) atomicAdd(&sm.bcast[0], v);
    __syncthreads();
    const int r = sm.bcast[0];
    __syncthreads();
    return r;
}

// The k largest keys (score image u descending, then index ascending) among the valid elements 0..n-1 of get(i, u):
// their keys go to keys[0..m) sorted descending, m = min(k, number valid) is returned.  `keys` (shared memory) holds the
// next power of two >= k keys: the bitonic sort pads to it.  An exact radix select of the
// k-th largest u (four 8-bit passes) gives the threshold T; every element above T is taken, and of those equal to T the
// ones with the smallest indices (an ordered scan).  Every thread calls it.
template <class Get>
__device__ int select_top_k(int n, int k, Get get, unsigned long long* keys, SelectScratch& sm) {
    const int tid = threadIdx.x;
    int local = 0;
    for (int i = tid; i < n; i += kDetThreads) {
        uint32_t u;
        local += get(i, u) ? 1 : 0;
    }
    const int valid = block_sum(local, sm);
    const bool all = valid <= k;
    uint32_t prefix = 0, mask = 0;
    int need = k;
    if (!all) {
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int b = tid; b < 256; b += kDetThreads) sm.hist[b] = 0;
            __syncthreads();
            for (int i = tid; i < n; i += kDetThreads) {
                uint32_t u;
                if (get(i, u) && (u & mask) == prefix) atomicAdd(&sm.hist[(u >> shift) & 255u], 1);
            }
            __syncthreads();
            if (tid == 0) {
                int acc = 0, b = 255;
                for (; b > 0; --b) {
                    if (acc + sm.hist[b] >= need) break;
                    acc += sm.hist[b];
                }
                sm.bcast[0] = b;
                sm.bcast[1] = need - acc;
            }
            __syncthreads();
            prefix |= static_cast<uint32_t>(sm.bcast[0]) << shift;
            mask |= 255u << shift;
            need = sm.bcast[1];
            __syncthreads();
        }
    }
    const int m = all ? valid : k;
    // compaction: above T, or the first `need` equal to T in index order
    if (tid == 0) sm.bcast[1] = 0;
    __syncthreads();
    int ties = 0;
    for (int base = 0; base < n; base += kDetThreads) {
        const int i = base + tid;
        uint32_t u = 0;
        const bool v = i < n && get(i, u);
        const bool eq = v && !all && u == prefix;
        int chunk_ties;
        const int before = block_scan(eq, &chunk_ties, sm);
        if (v && (all || u > prefix || (eq && ties + before < need))) keys[atomicAdd(&sm.bcast[1], 1)] = make_key(u, i);
        ties += chunk_ties;
    }
    // bitonic sort, descending, over the next power of two (padding keys 0 sort last: a real key is >= 1)
    int len = 1;
    while (len < m) len <<= 1;
    __syncthreads();
    for (int i = m + tid; i < len; i += kDetThreads) keys[i] = 0;
    __syncthreads();
    for (int size = 2; size <= len; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = tid; t < (len >> 1); t += kDetThreads) {
                const int lo = (t / stride) * stride * 2 + (t % stride), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const unsigned long long a = keys[lo], b = keys[hi];
                if (desc ? a < b : a > b) {
                    keys[lo] = b;
                    keys[hi] = a;
                }
            }
            __syncthreads();
        }
    return m;
}

// IoU of two boxes, operation by operation as include/fcuda.h states it (no contraction into FMA).  PLUS_ONE is
// Proposal's pixel convention: each side of the overlap is min - max + 1 (and the caller's areas carry the same + 1);
// without it the operations are DetectionOutput's and YOLO's.
template <bool PLUS_ONE = false>
__device__ __forceinline__ float box_iou(const float* a, float area_a, const float* b, float area_b) {
    float iw = __fsub_rn(fminf(a[2], b[2]), fmaxf(a[0], b[0]));
    float ih = __fsub_rn(fminf(a[3], b[3]), fmaxf(a[1], b[1]));
    if (PLUS_ONE) {
        iw = __fadd_rn(iw, 1.f);
        ih = __fadd_rn(ih, 1.f);
    }
    iw = fmaxf(iw, 0.f);
    ih = fmaxf(ih, 0.f);
    const float inter = __fmul_rn(iw, ih);
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

__global__ void __launch_bounds__(kDetThreads)
nms_class_kernel(const float* __restrict__ conf, const float* __restrict__ boxes, int P, int C, float conf_thr,
                 float nms_thr, int top_k, unsigned long long* __restrict__ kept, int* __restrict__ kept_count) {
    __shared__ SelectSmem sm;
    __shared__ float sb[kMaxTopK][4];
    __shared__ float sarea[kMaxTopK];
    __shared__ unsigned char sup[kMaxTopK];
    const int c = blockIdx.x, n = blockIdx.y;
    const int tid = threadIdx.x;
    const size_t list = static_cast<size_t>(n) * C + c;
    if (c == 0) {  // background
        if (tid == 0) kept_count[list] = 0;
        return;
    }
    const float* cf = conf + static_cast<size_t>(n) * P * C + c;
    const int m = select_top_k(P, top_k, [&](int i, uint32_t& u) {
        const float s = cf[static_cast<size_t>(i) * C];
        u = orderable(s);
        return s > conf_thr;
    }, sm.keys, sm.s);
    const float* ib = boxes + static_cast<size_t>(n) * P * 4;
    for (int j = tid; j < m; j += kDetThreads) {
        const float* b = ib + static_cast<size_t>(key_index(sm.keys[j])) * 4;
#pragma unroll
        for (int q = 0; q < 4; ++q) sb[j][q] = b[q];
        sarea[j] = __fmul_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1]));
        sup[j] = 0;
    }
    __syncthreads();
    for (int i = 0; i < m; ++i) {
        if (!sup[i])  // uniform: sup[i] was settled before the last barrier
            for (int j = i + 1 + tid; j < m; j += kDetThreads)
                if (!sup[j] && box_iou(sb[i], sarea[i], sb[j], sarea[j]) > nms_thr) sup[j] = 1;
        __syncthreads();
    }
    unsigned long long* out = kept + list * top_k;
    int written = 0;
    for (int base = 0; base < m; base += kDetThreads) {
        const int j = base + tid;
        const int keep = j < m && !sup[j];
        int total;
        const int pos = block_scan(keep, &total, sm.s);
        if (keep) out[written + pos] = sm.keys[j];
        written += total;
    }
    if (tid == 0) kept_count[list] = written;
}

__global__ void __launch_bounds__(kDetThreads)
merge_kernel(float* __restrict__ out, const float* __restrict__ conf, const float* __restrict__ boxes,
             const unsigned long long* __restrict__ kept, const int* __restrict__ kept_count, int P, int C, int top_k,
             int keep_top_k) {
    __shared__ SelectSmem sm;
    const int n = blockIdx.x;
    const unsigned long long* lists = kept + static_cast<size_t>(n) * C * top_k;
    const int* counts = kept_count + static_cast<size_t>(n) * C;
    // v = class * top_k + rank in that class's kept list: for equal scores, ascending v is (class, prior) ascending
    const int m = select_top_k(C * top_k, keep_top_k, [&](int v, uint32_t& u) {
        const int c = v / top_k;
        if (c == 0 || v - c * top_k >= counts[c]) return false;
        u = static_cast<uint32_t>(lists[v] >> 32);
        return true;
    }, sm.keys, sm.s);
    const float* ib = boxes + static_cast<size_t>(n) * P * 4;
    float* o = out + static_cast<size_t>(n) * keep_top_k * 6;
    for (int r = threadIdx.x; r < keep_top_k; r += kDetThreads) {
        float* row = o + static_cast<size_t>(r) * 6;
        if (r < m) {
            const int v = key_index(sm.keys[r]);
            const int c = v / top_k, prior = key_index(lists[v]);
            const float* b = ib + static_cast<size_t>(prior) * 4;
            row[0] = static_cast<float>(c);
            row[1] = conf[(static_cast<size_t>(n) * P + prior) * C + c];
            row[2] = b[0];
            row[3] = b[1];
            row[4] = b[2];
            row[5] = b[3];
        } else {
            row[0] = -1.f;
            row[1] = row[2] = row[3] = row[4] = row[5] = 0.f;
        }
    }
}

struct DetWorkspace {
    float* boxes;
    unsigned long long* kept;
    int* counts;
};

DetWorkspace carve(float* ws, int P, int C, int top_k, int batch) {
    DetWorkspace w;
    const size_t box_floats = round_up_sz(static_cast<size_t>(batch) * P * 4, 4);
    const size_t kept_floats = static_cast<size_t>(batch) * C * top_k * 2;
    w.boxes = ws;
    w.kept = reinterpret_cast<unsigned long long*>(ws + box_floats);
    w.counts = reinterpret_cast<int*>(ws + box_floats + kept_floats);
    return w;
}

// ---- YOLO (YoloDetectionOutput, Yolov3DetectionOutput) --------------------------------------------------------------
// decode  one thread per (image, slot): confidence, class and box of every slot;
// select  one CTA per image: select_top_k over the candidates (score >= threshold), their sorted keys, boxes and areas;
// mask    CTAs over (32-row block, image): word w of row i has bit b set iff j = 32 w + b > i and IoU(i, j) > threshold;
// sweep   one CTA per image: the mask in shared memory, one warp walks the candidates in order (lane l owns the removal
//         word l: no barrier and no global load in the loop), then the output rows.
constexpr int kYoloMaskWords = kMaxTopK / 32;
constexpr int kYoloMaskRows = 32;  // rows of one mask CTA: 8 warps x 4

// Per-scale geometry, by value: the bottom, its grid, its first slot and, per box, the anchor and its normaliser
// (version 3: (int)(anchors_scale * w); version 2: the grid side).
struct YoloScale {
    const float* in;
    int h, w, slot0;
    float norm_w, norm_h;
    float bias_w[FCUDA_YOLO_MAX_BOXES], bias_h[FCUDA_YOLO_MAX_BOXES];
};
struct YoloGeom {
    int version, num_class, num_box, num_scales, slots;
    YoloScale scale[FCUDA_YOLO_MAX_SCALES];
};

__global__ void __launch_bounds__(256)
yolo_decode_kernel(float* __restrict__ scores, int* __restrict__ classes, float* __restrict__ boxes, const YoloGeom g,
                   long long total) {
    const int stride = 5 + g.num_class;
    for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
         t += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long n = t / g.slots;
        const int slot = static_cast<int>(t - n * g.slots);
        int b = 0;
        while (b + 1 < g.num_scales && slot >= g.scale[b + 1].slot0) ++b;
        const YoloScale& sc = g.scale[b];
        const int hw = sc.h * sc.w;
        const int r = slot - sc.slot0, pp = r / hw, cell = r - pp * hw;
        const int i = cell / sc.w, j = cell - i * sc.w;
        const float* p = sc.in + (static_cast<size_t>(n) * g.num_box + pp) * stride * hw + cell;
        const float tx = p[0], ty = p[static_cast<size_t>(hw)], tw = p[2 * static_cast<size_t>(hw)];
        const float th = p[3 * static_cast<size_t>(hw)], obj = p[4 * static_cast<size_t>(hw)];
        const float* logit = p + 5 * static_cast<size_t>(hw);
        int cls = 0;
        float conf;
        if (g.version == 3) {
            float m = -FLT_MAX;
            for (int k = 0; k < g.num_class; ++k) {
                const float v = logit[static_cast<size_t>(k) * hw];
                if (v > m) {
                    m = v;
                    cls = k;
                }
            }
            conf = __fdiv_rn(1.f, __fadd_rn(1.f, __fmul_rn(expf(-obj), __fadd_rn(1.f, expf(-m)))));
        } else {
            float m = -FLT_MAX;  // ncnn's Softmax: a NaN logit does not become the max
            for (int k = 0; k < g.num_class; ++k) m = fmaxf(m, logit[static_cast<size_t>(k) * hw]);
            float sum = 0.f;
            for (int k = 0; k < g.num_class; ++k) sum = __fadd_rn(sum, expf(__fsub_rn(logit[static_cast<size_t>(k) * hw], m)));
            float best = 0.f;
            for (int k = 0; k < g.num_class; ++k) {
                const float pk = __fdiv_rn(expf(__fsub_rn(logit[static_cast<size_t>(k) * hw], m)), sum);
                if (pk > best) {
                    best = pk;
                    cls = k;
                }
            }
            conf = __fmul_rn(sigm(obj), best);
        }
        const float cx = __fdiv_rn(__fadd_rn(static_cast<float>(j), sigm(tx)), static_cast<float>(sc.w));
        const float cy = __fdiv_rn(__fadd_rn(static_cast<float>(i), sigm(ty)), static_cast<float>(sc.h));
        const float bw = __fdiv_rn(__fmul_rn(expf(tw), sc.bias_w[pp]), sc.norm_w);
        const float bh = __fdiv_rn(__fmul_rn(expf(th), sc.bias_h[pp]), sc.norm_h);
        scores[t] = conf;
        classes[t] = cls;
        float* o = boxes + static_cast<size_t>(t) * 4;
        o[0] = __fsub_rn(cx, __fmul_rn(bw, 0.5f));
        o[1] = __fsub_rn(cy, __fmul_rn(bh, 0.5f));
        o[2] = __fadd_rn(cx, __fmul_rn(bw, 0.5f));
        o[3] = __fadd_rn(cy, __fmul_rn(bh, 0.5f));
    }
}

struct YoloWorkspace {
    unsigned long long* keys;  // (batch, kMaxTopK)
    uint32_t* mask;            // (batch, kMaxTopK, kYoloMaskWords)
    float* sel_box;            // (batch, kMaxTopK, 4)
    float* sel_area;           // (batch, kMaxTopK)
    float* boxes;              // (batch, slots, 4)
    float* scores;             // (batch, slots)
    int* classes;              // (batch, slots)
    int* counts;               // (batch)
};

YoloWorkspace yolo_carve(float* ws, int slots, int batch) {
    YoloWorkspace w;
    const size_t n = static_cast<size_t>(batch);
    w.keys = reinterpret_cast<unsigned long long*>(ws);
    ws += n * kMaxTopK * 2;
    w.mask = reinterpret_cast<uint32_t*>(ws);
    ws += n * kMaxTopK * kYoloMaskWords;
    w.sel_box = ws;
    ws += n * kMaxTopK * 4;
    w.sel_area = ws;
    ws += n * kMaxTopK;
    w.boxes = ws;
    ws += n * slots * 4;
    w.scores = ws;
    ws += n * slots;
    w.classes = reinterpret_cast<int*>(ws);
    ws += n * slots;
    w.counts = reinterpret_cast<int*>(ws);
    return w;
}

__global__ void __launch_bounds__(kDetThreads)
yolo_select_kernel(const YoloWorkspace w, int slots, float thr, int top_k) {
    __shared__ SelectSmem sm;
    const int n = blockIdx.x;
    const float* sc = w.scores + static_cast<size_t>(n) * slots;
    const int m = select_top_k(slots, top_k, [&](int i, uint32_t& u) {
        const float s = sc[i];
        u = orderable(s);
        return s >= thr;
    }, sm.keys, sm.s);
    const float* ib = w.boxes + static_cast<size_t>(n) * slots * 4;
    for (int j = threadIdx.x; j < m; j += kDetThreads) {
        const unsigned long long key = sm.keys[j];
        const float* b = ib + static_cast<size_t>(key_index(key)) * 4;
        float* o = w.sel_box + (static_cast<size_t>(n) * kMaxTopK + j) * 4;
#pragma unroll
        for (int q = 0; q < 4; ++q) o[q] = b[q];
        w.sel_area[static_cast<size_t>(n) * kMaxTopK + j] = __fmul_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1]));
        w.keys[static_cast<size_t>(n) * kMaxTopK + j] = key;
    }
    if (threadIdx.x == 0) w.counts[n] = m;
}

// Row i of the suppression mask over m candidates staged in sb / sarea: every lane of the warp calls it and gets word
// `lane` (bit b set iff j = 32 lane + b > i and IoU(i, j) > nms_thr).
__device__ __forceinline__ uint32_t yolo_mask_row(int i, int m, const float (*sb)[4], const float* sarea, float nms_thr,
                                                  int lane) {
    uint32_t mine = 0;
    const int words = (m + 31) >> 5;
    for (int wd = i >> 5; wd < words; ++wd) {
        const int j = (wd << 5) + lane;
        const bool hit = j > i && j < m && box_iou(sb[i], sarea[i], sb[j], sarea[j]) > nms_thr;
        const uint32_t bits = __ballot_sync(0xffffffffu, hit);
        if (lane == wd) mine = bits;
    }
    return mine;
}

// Stage the selected boxes and areas j in [from, m) of image n.  The caller synchronises.
__device__ __forceinline__ void yolo_stage_boxes(const YoloWorkspace& w, int n, int from, int m, float (*sb)[4],
                                                 float* sarea) {
    const float* gb = w.sel_box + static_cast<size_t>(n) * kMaxTopK * 4;
    const float* ga = w.sel_area + static_cast<size_t>(n) * kMaxTopK;
    for (int j = from + threadIdx.x; j < m; j += blockDim.x) {
#pragma unroll
        for (int q = 0; q < 4; ++q) sb[j][q] = gb[static_cast<size_t>(j) * 4 + q];
        sarea[j] = ga[j];
    }
}

// The greedy walk over the shared-memory mask (m rows of kYoloMaskWords words) and the output rows of image n.  One warp
// walks the candidates in order, lane l owning removal word l: no barrier and no global load in the loop; it stops at
// keep_top_k kept boxes.  Every thread of the CTA calls it.
__device__ __forceinline__ void yolo_sweep_rows(float* __restrict__ out, const YoloWorkspace& w, int n, int m, int slots,
                                                int keep_top_k, const uint32_t* smask, int* keep, int* kept_count) {
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        uint32_t removed = 0;  // lane l: candidates 32 l .. 32 l + 31 suppressed by a kept box
        int kept = 0;
        for (int i = 0; i < m && kept < keep_top_k; ++i) {
            const uint32_t word = __shfl_sync(0xffffffffu, removed, i >> 5);
            if (!((word >> (i & 31)) & 1u)) {  // uniform over the warp
                if (lane == 0) keep[kept] = i;
                ++kept;
                removed |= smask[i * kYoloMaskWords + lane];
            }
        }
        if (lane == 0) *kept_count = kept;
    }
    __syncthreads();
    const int kept = *kept_count;
    const unsigned long long* keys = w.keys + static_cast<size_t>(n) * kMaxTopK;
    const float* sel = w.sel_box + static_cast<size_t>(n) * kMaxTopK * 4;
    float* o = out + static_cast<size_t>(n) * keep_top_k * 6;
    for (int r = threadIdx.x; r < keep_top_k; r += blockDim.x) {
        float* row = o + static_cast<size_t>(r) * 6;
        if (r < kept) {
            const int c = keep[r];
            const size_t slot = static_cast<size_t>(n) * slots + key_index(keys[c]);
            row[0] = static_cast<float>(w.classes[slot] + 1);
            row[1] = w.scores[slot];
#pragma unroll
            for (int q = 0; q < 4; ++q) row[2 + q] = sel[static_cast<size_t>(c) * 4 + q];
        } else {
            row[0] = -1.f;
            row[1] = row[2] = row[3] = row[4] = row[5] = 0.f;
        }
    }
}

// Split NMS, first half: CTAs over (32-row block, image) write the mask to the workspace.
__global__ void __launch_bounds__(256)
yolo_mask_kernel(const YoloWorkspace w, float nms_thr) {
    __shared__ float sb[kMaxTopK][4];
    __shared__ float sarea[kMaxTopK];
    const int n = blockIdx.y, row0 = blockIdx.x * kYoloMaskRows;
    const int m = w.counts[n];
    if (row0 >= m) return;
    yolo_stage_boxes(w, n, row0, m, sb, sarea);  // only columns >= row0 can be set
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* out = w.mask + static_cast<size_t>(n) * kMaxTopK * kYoloMaskWords;
    for (int i = row0 + warp; i < row0 + kYoloMaskRows && i < m; i += 8)
        out[static_cast<size_t>(i) * kYoloMaskWords + lane] = yolo_mask_row(i, m, sb, sarea, nms_thr, lane);
}

// Split NMS, second half: one CTA per image stages the mask (16-byte loads: the workspace is 16-byte aligned and every
// offset into it is a multiple of 16 bytes) and sweeps it.
__global__ void __launch_bounds__(kDetThreads)
yolo_sweep_kernel(float* __restrict__ out, const YoloWorkspace w, int slots, int keep_top_k) {
    extern __shared__ uint4 yolo_smem[];
    __shared__ int keep[kMaxTopK];
    __shared__ int kept_count;
    const int n = blockIdx.x;
    const int m = w.counts[n];
    const uint4* gm = reinterpret_cast<const uint4*>(w.mask + static_cast<size_t>(n) * kMaxTopK * kYoloMaskWords);
    for (int v = threadIdx.x; v < m * (kYoloMaskWords / 4); v += kDetThreads) yolo_smem[v] = gm[v];
    __syncthreads();
    yolo_sweep_rows(out, w, n, m, slots, keep_top_k, reinterpret_cast<const uint32_t*>(yolo_smem), keep, &kept_count);
}

}  // namespace

int permute_forward(const float* in, float* out, int c, int h, int w, int order, int batch, cudaStream_t s) {
    const long long total = static_cast<long long>(batch) * c * h * w;
    const int prof = prof_begin(s, PROF_DETECTION, 0, 0, 8.0 * total);
    if (order == 0) {
        FCUDA_CHECK(cudaMemcpyAsync(out, in, static_cast<size_t>(total) * sizeof(float), cudaMemcpyDeviceToDevice, s));
    } else if (order == 3 && batch <= 65535) {
        const int rows = c, cols = h * w;
        const dim3 grid(static_cast<unsigned>(ceil_div(cols, kTile)), static_cast<unsigned>(ceil_div(rows, kTile)),
                        static_cast<unsigned>(batch));
        transpose_kernel<<<grid, dim3(kTile, 8), 0, s>>>(in, out, rows, cols);
        FCUDA_CHECK_LAUNCH();
    } else {
        const long long blocks = (total + 255) / 256;
        permute_kernel<<<static_cast<unsigned>(blocks < 65536 * 4 ? blocks : 65536 * 4), 256, 0, s>>>(in, out, c, h, w, order,
                                                                                                       total);
        FCUDA_CHECK_LAUNCH();
    }
    prof_end(prof, s);
    count_launch();
    return 0;
}

int softmax_axis_forward(const float* in, float* out, int outer, int len, int inner, int batch, cudaStream_t s) {
    const long long lines = static_cast<long long>(batch) * outer * inner;
    const int prof = prof_begin(s, PROF_DETECTION, 0, 0, 8.0 * lines * len);
    if (inner == 1) {
        const long long blocks = (lines + 7) / 8;
        if (blocks > 0x7fffffffLL) return -100;
        softmax_rows_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(in, out, lines, len);
    } else {
        const long long blocks = (lines + 255) / 256;
        if (blocks > 0x7fffffffLL) return -100;
        softmax_cols_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(in, out, lines, len, inner);
    }
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

int priorbox_forward(float* out, const FcudaPriorBoxParam& p, int per_loc, int feat_w, int feat_h, float img_w, float img_h,
                     float step_w, float step_h, cudaStream_t s) {
    const int locs = feat_w * feat_h;
    const int prof = prof_begin(s, PROF_DETECTION, 0, 0, 32.0 * locs * per_loc);
    priorbox_kernel<<<static_cast<unsigned>(ceil_div(locs, 256)), 256, 0, s>>>(out, p, per_loc, feat_w, feat_h, img_w, img_h,
                                                                              step_w, step_h);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

int ssd_decode(float* boxes, const float* loc, const float* priors, int num_priors, int batch, cudaStream_t s) {
    const long long total = static_cast<long long>(batch) * num_priors;
    const int prof = prof_begin(s, PROF_DETECTION, 0, 0, 32.0 * total + 32.0 * num_priors);
    decode_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(boxes, loc, priors, num_priors, total);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

size_t detection_output_workspace(int num_priors, int num_classes, int nms_top_k, int batch) {
    return round_up_sz(static_cast<size_t>(batch) * num_priors * 4, 4) + static_cast<size_t>(batch) * num_classes * nms_top_k * 2 +
           static_cast<size_t>(batch) * num_classes;
}

int detection_output(float* out, const float* loc, const float* conf, const float* priors, int P, int C, float conf_threshold,
                     float nms_threshold, int nms_top_k, int keep_top_k, float* workspace, int batch, cudaStream_t s) {
    const DetWorkspace w = carve(workspace, P, C, nms_top_k, batch);
    int rc = ssd_decode(w.boxes, loc, priors, P, batch, s);
    if (rc) return rc;
    const double scores = static_cast<double>(batch) * P * C;
    int prof = prof_begin(s, PROF_DETECTION, 0, 0, 4.0 * scores + 16.0 * batch * P);
    nms_class_kernel<<<dim3(static_cast<unsigned>(C), static_cast<unsigned>(batch)), kDetThreads, 0, s>>>(
        conf, w.boxes, P, C, conf_threshold, nms_threshold, nms_top_k, w.kept, w.counts);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    prof = prof_begin(s, PROF_DETECTION, 0, 0, 24.0 * batch * keep_top_k);
    merge_kernel<<<static_cast<unsigned>(batch), kDetThreads, 0, s>>>(out, conf, w.boxes, w.kept, w.counts, P, C,
                                                                       nms_top_k, keep_top_k);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

namespace {

YoloGeom yolo_geom(const float* const* inputs, const FcudaYoloParam& p) {
    YoloGeom g{};
    g.version = p.version;
    g.num_class = p.num_class;
    g.num_box = p.num_box;
    g.num_scales = p.num_scales;
    int slot0 = 0;
    for (int b = 0; b < p.num_scales; ++b) {
        YoloScale& sc = g.scale[b];
        sc.in = inputs[b];
        sc.h = p.grid_h[b];
        sc.w = p.grid_w[b];
        sc.slot0 = slot0;
        slot0 += p.num_box * sc.h * sc.w;
        if (p.version == 3) {
            sc.norm_w = static_cast<float>(static_cast<int>(p.anchors_scale[b] * static_cast<float>(sc.w)));
            sc.norm_h = static_cast<float>(static_cast<int>(p.anchors_scale[b] * static_cast<float>(sc.h)));
        } else {
            sc.norm_w = static_cast<float>(sc.w);
            sc.norm_h = static_cast<float>(sc.h);
        }
        for (int pp = 0; pp < p.num_box; ++pp) {
            const int k = p.version == 3 ? p.mask[b * p.num_box + pp] : pp;
            sc.bias_w[pp] = p.biases[2 * k];
            sc.bias_h[pp] = p.biases[2 * k + 1];
        }
    }
    g.slots = slot0;
    return g;
}

int yolo_decode_launch(float* scores, int* classes, float* boxes, const YoloGeom& g, int batch, cudaStream_t s) {
    const long long total = static_cast<long long>(batch) * g.slots;
    const int prof = prof_begin(s, PROF_DETECTION, 0, 0, 4.0 * (5 + g.num_class) * total + 24.0 * total);
    const long long blocks = (total + 255) / 256;
    yolo_decode_kernel<<<static_cast<unsigned>(blocks < 65536 * 16 ? blocks : 65536 * 16), 256, 0, s>>>(scores, classes,
                                                                                                        boxes, g, total);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

SmemAttrCache yolo_sweep_smem;

}  // namespace

int yolo_decode(float* scores, int* classes, float* boxes, const float* const* inputs, const FcudaYoloParam& p, int batch,
                cudaStream_t s) {
    return yolo_decode_launch(scores, classes, boxes, yolo_geom(inputs, p), batch, s);
}

size_t yolo_detection_workspace(int slots, int batch) {
    return static_cast<size_t>(batch) * (6 * static_cast<size_t>(slots) + 2 * kMaxTopK + kMaxTopK * kYoloMaskWords +
                                         5 * kMaxTopK + 1);
}

int yolo_detection(float* out, const float* const* inputs, const FcudaYoloParam& p, float* workspace, int batch,
                   cudaStream_t s) {
    const YoloGeom g = yolo_geom(inputs, p);
    const YoloWorkspace w = yolo_carve(workspace, g.slots, batch);
    int rc = yolo_decode_launch(w.scores, w.classes, w.boxes, g, batch, s);
    if (rc) return rc;
    const double slots = static_cast<double>(batch) * g.slots;
    int prof = prof_begin(s, PROF_DETECTION, 0, 0, 4.0 * slots + 24.0 * batch * p.nms_top_k);
    yolo_select_kernel<<<static_cast<unsigned>(batch), kDetThreads, 0, s>>>(w, g.slots, p.confidence_threshold,
                                                                             p.nms_top_k);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    const int smem = p.nms_top_k * kYoloMaskWords * static_cast<int>(sizeof(uint32_t));
    const int row_blocks = ceil_div(p.nms_top_k, kYoloMaskRows);
    prof = prof_begin(s, PROF_DETECTION, 0, 0, 20.0 * batch * p.nms_top_k + 4.0 * batch * p.nms_top_k * kYoloMaskWords);
    yolo_mask_kernel<<<dim3(static_cast<unsigned>(row_blocks), static_cast<unsigned>(batch)), 256, 0, s>>>(w,
                                                                                                        p.nms_threshold);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    rc = ensure_dynamic_smem(yolo_sweep_kernel, smem, yolo_sweep_smem);
    if (rc) return rc;
    prof = prof_begin(s, PROF_DETECTION, 0, 0, 4.0 * batch * p.nms_top_k * kYoloMaskWords + 24.0 * batch * p.keep_top_k);
    yolo_sweep_kernel<<<static_cast<unsigned>(batch), kDetThreads, smem, s>>>(out, w, g.slots, p.keep_top_k);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

namespace {

// ---- Faster R-CNN: Proposal and ROIPooling -------------------------------------------------------------------------
// decode    one thread per (image, anchor, cell): the clipped box and the candidate key (the orderable image of the
//           foreground score, 0 for a box below min_size or a NaN score) into the workspace;
// select    one CTA per image: select_top_k over the A * H * W keys, up to kProposalMaxTopK of them sorted in dynamic
//           shared memory; the selected boxes, their + 1 areas and anchor-cell indices go to the workspace;
// mask      CTAs over (32-row block, image): word w of row i has bit b set iff j = 32 w + b > i and IoU(i, j) > thresh,
//           the columns staged through shared memory 1024 at a time; K x ceil(K / 32) words in global memory;
// sweep     one warp per image: the removal bitmap in shared memory; find-first-set over the live bits of one word at a
//           time, each kept box ORs its mask row (from L2) into the bitmap and writes its output row; stops at
//           after_nms_topN.
// roi_pool  one thread per output element, pooled x fastest.
// psroi     R-FCN's position-sensitive average pooling: one thread per output element, pooled x fastest; bin (ph, pw) of
//           output channel q reads input channel (q * PH + ph) * PW + pw.
constexpr int kProposalAnchors = 9;  // ratios {0.5, 1, 2} x scales {8, 16, 32}
constexpr int kMaskChunk = 1024;     // columns of the mask staged per pass

struct ProposalGeom {
    int A, H, W, P;  // anchors, feature map, A * H * W
    float stride, min_size;
    float ax1[kProposalAnchors], ay1[kProposalAnchors], aw[kProposalAnchors], ah[kProposalAnchors];
};

struct ProposalWorkspace {
    float* boxes;     // (batch, P, 4) clipped boxes
    uint32_t* keys;   // (batch, P4) orderable score, 0 = not a candidate
    float* sel_box;   // (batch, K, 4)
    float* sel_area;  // (batch, K4)
    int* sel_idx;     // (batch, K4)
    int* counts;      // (batch4)
    uint32_t* mask;   // (batch, K, words)
    int P4, K, K4, words;
};

size_t round4(size_t v) { return round_up_sz(v, 4); }

ProposalWorkspace proposal_carve(float* ws, int P, int K, int batch) {
    ProposalWorkspace w;
    const size_t n = static_cast<size_t>(batch);
    w.P4 = static_cast<int>(round4(P));
    w.K = K;
    w.K4 = static_cast<int>(round4(K));
    w.words = ceil_div(K, 32);
    w.boxes = ws;
    ws += n * P * 4;
    w.keys = reinterpret_cast<uint32_t*>(ws);
    ws += n * w.P4;
    w.sel_box = ws;
    ws += n * K * 4;
    w.sel_area = ws;
    ws += n * w.K4;
    w.sel_idx = reinterpret_cast<int*>(ws);
    ws += n * w.K4;
    w.counts = reinterpret_cast<int*>(ws);
    ws += round4(n);
    w.mask = reinterpret_cast<uint32_t*>(ws);
    return w;
}

// boxes: (batch, P, 4); keys: (batch, key_stride) or null (decode alone)
__global__ void __launch_bounds__(256)
proposal_decode_kernel(float4* __restrict__ boxes, uint32_t* __restrict__ keys, int key_stride,
                       const float* __restrict__ score, const float* __restrict__ bbox, const float* __restrict__ im_info,
                       const ProposalGeom g, long long total) {
    const int hw = g.H * g.W;
    for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
         t += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long n = t / g.P;
        const int i = static_cast<int>(t - n * g.P);
        const int q = i / hw, cell = i - q * hw;
        const int y = cell / g.W, x = cell - y * g.W;
        const float* d = bbox + (static_cast<size_t>(n) * 4 * g.A + 4 * q) * hw + cell;
        const float dx = d[0], dy = d[static_cast<size_t>(hw)], dw = d[2 * static_cast<size_t>(hw)];
        const float dh = d[3 * static_cast<size_t>(hw)];
        const float aw = g.aw[q], ah = g.ah[q];
        const float ax = __fadd_rn(g.ax1[q], __fmul_rn(static_cast<float>(x), g.stride));
        const float ay = __fadd_rn(g.ay1[q], __fmul_rn(static_cast<float>(y), g.stride));
        const float pcx = __fadd_rn(__fadd_rn(ax, __fmul_rn(aw, 0.5f)), __fmul_rn(aw, dx));
        const float pcy = __fadd_rn(__fadd_rn(ay, __fmul_rn(ah, 0.5f)), __fmul_rn(ah, dy));
        const float pw = __fmul_rn(aw, expf(dw)), ph = __fmul_rn(ah, expf(dh));
        const float* info = im_info + static_cast<size_t>(n) * 3;
        const float xmax = __fsub_rn(info[1], 1.f), ymax = __fsub_rn(info[0], 1.f);
        float4 b;
        b.x = fmaxf(fminf(__fsub_rn(pcx, __fmul_rn(pw, 0.5f)), xmax), 0.f);
        b.y = fmaxf(fminf(__fsub_rn(pcy, __fmul_rn(ph, 0.5f)), ymax), 0.f);
        b.z = fmaxf(fminf(__fadd_rn(pcx, __fmul_rn(pw, 0.5f)), xmax), 0.f);
        b.w = fmaxf(fminf(__fadd_rn(pcy, __fmul_rn(ph, 0.5f)), ymax), 0.f);
        boxes[t] = b;
        if (keys) {
            const float s = score[(static_cast<size_t>(n) * 2 * g.A + g.A + q) * hw + cell];
            const float thr = __fmul_rn(g.min_size, info[2]);
            const bool ok = !isnan(s) && __fadd_rn(__fsub_rn(b.z, b.x), 1.f) >= thr &&
                            __fadd_rn(__fsub_rn(b.w, b.y), 1.f) >= thr;
            keys[static_cast<size_t>(n) * key_stride + i] = ok ? orderable(s) : 0u;  // a non-NaN image is never 0
        }
    }
}

__device__ __forceinline__ float area_plus_one(float4 b) {
    return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
}

__global__ void __launch_bounds__(kDetThreads)
proposal_select_kernel(const ProposalWorkspace w, int P) {
    extern __shared__ unsigned long long proposal_keys[];
    __shared__ SelectScratch sm;
    const int n = blockIdx.x;
    const uint32_t* ku = w.keys + static_cast<size_t>(n) * w.P4;
    const int m = select_top_k(P, w.K, [&](int i, uint32_t& u) {
        u = ku[i];
        return u != 0u;
    }, proposal_keys, sm);
    const float4* ib = reinterpret_cast<const float4*>(w.boxes) + static_cast<size_t>(n) * P;
    float4* ob = reinterpret_cast<float4*>(w.sel_box) + static_cast<size_t>(n) * w.K;
    for (int j = threadIdx.x; j < m; j += kDetThreads) {
        const int idx = key_index(proposal_keys[j]);
        const float4 b = ib[idx];
        ob[j] = b;
        w.sel_area[static_cast<size_t>(n) * w.K4 + j] = area_plus_one(b);
        w.sel_idx[static_cast<size_t>(n) * w.K4 + j] = idx;
    }
    if (threadIdx.x == 0) w.counts[n] = m;
}

// 8 warps x 4 rows; every row's words from its own word on, a chunk of 32 words (1024 columns) per staging pass
__global__ void __launch_bounds__(256)
proposal_mask_kernel(const ProposalWorkspace w, float nms_thr) {
    __shared__ float4 sb[kMaskChunk];
    __shared__ float sa[kMaskChunk];
    const int n = blockIdx.y, row0 = blockIdx.x * 32;
    const int m = w.counts[n];
    if (row0 >= m) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int words = (m + 31) >> 5;
    const float4* gb = reinterpret_cast<const float4*>(w.sel_box) + static_cast<size_t>(n) * w.K;
    const float* ga = w.sel_area + static_cast<size_t>(n) * w.K4;
    float rb[4][4], ra[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int i = min(row0 + warp + 8 * r, m - 1);
        const float4 b = gb[i];
        rb[r][0] = b.x;
        rb[r][1] = b.y;
        rb[r][2] = b.z;
        rb[r][3] = b.w;
        ra[r] = ga[i];
    }
    uint32_t* out = w.mask + static_cast<size_t>(n) * w.K * w.words;
    for (int c0 = row0; c0 < m; c0 += kMaskChunk) {  // row0 is a multiple of 32: chunks start on a word
        const int cn = min(kMaskChunk, m - c0);
        __syncthreads();
        for (int j = threadIdx.x; j < cn; j += blockDim.x) {
            sb[j] = gb[c0 + j];
            sa[j] = ga[c0 + j];
        }
        __syncthreads();
        const int w0 = c0 >> 5, nw = min(32, words - w0);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int i = row0 + warp + 8 * r;
            if (i >= m) break;  // uniform over the warp
            uint32_t mine = 0;
            for (int k = 0; k < nw; ++k) {
                const int j = c0 + 32 * k + lane;
                if (c0 + 32 * k + 31 <= i) continue;  // the whole word is at or before row i: never read
                const bool hit = j > i && j < m &&
                                 box_iou<true>(rb[r], ra[r], reinterpret_cast<const float*>(&sb[j - c0]), sa[j - c0]) >
                                     nms_thr;
                const uint32_t bits = __ballot_sync(0xffffffffu, hit);
                if (lane == k) mine = bits;
            }
            if (lane < nw && w0 + lane >= (i >> 5)) out[static_cast<size_t>(i) * w.words + w0 + lane] = mine;
        }
    }
}

// rois: (batch, post, 4); scores: (batch, post) or null
__global__ void __launch_bounds__(32)
proposal_sweep_kernel(float4* __restrict__ rois, float* __restrict__ scores, const float* __restrict__ score,
                      const ProposalWorkspace w, int A, int hw, int post) {
    __shared__ uint32_t removed[kProposalMaxTopK / 32];
    const int n = blockIdx.x, lane = threadIdx.x;
    const int m = w.counts[n];
    const int words = (m + 31) >> 5;
    for (int v = lane; v < words; v += 32) removed[v] = 0u;
    __syncwarp();
    const float4* sel = reinterpret_cast<const float4*>(w.sel_box) + static_cast<size_t>(n) * w.K;
    const int* sel_idx = w.sel_idx + static_cast<size_t>(n) * w.K4;
    const uint32_t* mask = w.mask + static_cast<size_t>(n) * w.K * w.words;
    const float* fg = score + (static_cast<size_t>(n) * 2 * A + A) * hw;
    float4* orow = rois + static_cast<size_t>(n) * post;
    float* srow = scores ? scores + static_cast<size_t>(n) * post : nullptr;
    int kept = 0;
    for (int wd = 0; wd < words && kept < post; ++wd) {
        const uint32_t valid = (wd == words - 1 && (m & 31)) ? (1u << (m & 31)) - 1u : 0xffffffffu;
        uint32_t live = ~removed[wd] & valid;
        while (live && kept < post) {  // uniform: every lane reads the same words
            const int b = __ffs(live) - 1, i = (wd << 5) + b;
            if (lane == 0) {
                orow[kept] = sel[i];
                if (srow) srow[kept] = fg[sel_idx[i]];
            }
            ++kept;
            const uint32_t* row = mask + static_cast<size_t>(i) * w.words;
            for (int v = wd + lane; v < words; v += 32) removed[v] |= row[v];
            __syncwarp();
            live = ~removed[wd] & valid & (b == 31 ? 0u : 0xffffffffu << (b + 1));
        }
    }
    for (int r = kept + lane; r < post; r += 32) {
        orow[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (srow) srow[r] = -1.f;
    }
}

__global__ void __launch_bounds__(256)
roi_pool_kernel(float* __restrict__ out, const float* __restrict__ in, const float* __restrict__ rois, int C, int H,
                int W, int R, int PH, int PW, float scale, long long total) {
    for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
         t += static_cast<long long>(gridDim.x) * blockDim.x) {
        long long r = t;
        const int pw = static_cast<int>(r % PW);
        r /= PW;
        const int ph = static_cast<int>(r % PH);
        r /= PH;
        const int c = static_cast<int>(r % C);
        const long long item = r / C, n = item / R;
        const float* roi = rois + item * 4;
        // (int)roundf: half away from zero, converted saturating (a NaN corner reads as 0)
        const long long x1 = static_cast<int>(roundf(__fmul_rn(roi[0], scale)));
        const long long y1 = static_cast<int>(roundf(__fmul_rn(roi[1], scale)));
        const long long x2 = static_cast<int>(roundf(__fmul_rn(roi[2], scale)));
        const long long y2 = static_cast<int>(roundf(__fmul_rn(roi[3], scale)));
        const long long rw = max(x2 - x1 + 1, 1ll), rh = max(y2 - y1 + 1, 1ll);
        const float bin_w = __fdiv_rn(static_cast<float>(rw), static_cast<float>(PW));
        const float bin_h = __fdiv_rn(static_cast<float>(rh), static_cast<float>(PH));
        const long long ws = min(max(static_cast<long long>(floorf(__fmul_rn(static_cast<float>(pw), bin_w))) + x1, 0ll),
                                 static_cast<long long>(W));
        const long long we = min(max(static_cast<long long>(ceilf(__fmul_rn(static_cast<float>(pw + 1), bin_w))) + x1, 0ll),
                                 static_cast<long long>(W));
        const long long hs = min(max(static_cast<long long>(floorf(__fmul_rn(static_cast<float>(ph), bin_h))) + y1, 0ll),
                                 static_cast<long long>(H));
        const long long he = min(max(static_cast<long long>(ceilf(__fmul_rn(static_cast<float>(ph + 1), bin_h))) + y1, 0ll),
                                 static_cast<long long>(H));
        float v = 0.f;
        if (we > ws && he > hs) {
            const float* plane = in + (static_cast<size_t>(n) * C + c) * H * W;
            v = -FLT_MAX;
            for (long long h = hs; h < he; ++h)
                for (long long x = ws; x < we; ++x) v = fmaxf(v, __ldg(plane + h * W + x));
        }
        out[t] = v;
    }
}

// (int)floorf / ceilf converted saturating (a NaN reads as 0), then clamped to [0, hi]
__device__ __forceinline__ int psroi_edge(float v, int hi) { return min(max(static_cast<int>(v), 0), hi); }

__global__ void __launch_bounds__(256)
psroi_pool_kernel(float* __restrict__ out, const float* __restrict__ in, const float* __restrict__ rois, int C, int H,
                  int W, int R, int PH, int PW, int D, float scale, long long total) {
    for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
         t += static_cast<long long>(gridDim.x) * blockDim.x) {
        long long r = t;
        const int pw = static_cast<int>(r % PW);
        r /= PW;
        const int ph = static_cast<int>(r % PH);
        r /= PH;
        const int q = static_cast<int>(r % D);
        const long long item = r / D, n = item / R;
        const float* roi = rois + item * 4;
        const float x1 = __fmul_rn(roundf(roi[0]), scale), y1 = __fmul_rn(roundf(roi[1]), scale);
        const float x2 = __fmul_rn(roundf(__fadd_rn(roi[2], 1.f)), scale);
        const float y2 = __fmul_rn(roundf(__fadd_rn(roi[3], 1.f)), scale);
        const float bin_w = __fdiv_rn(fmaxf(__fsub_rn(x2, x1), 0.1f), static_cast<float>(PW));
        const float bin_h = __fdiv_rn(fmaxf(__fsub_rn(y2, y1), 0.1f), static_cast<float>(PH));
        const int ws = psroi_edge(floorf(__fadd_rn(x1, __fmul_rn(static_cast<float>(pw), bin_w))), W);
        const int we = psroi_edge(ceilf(__fadd_rn(x1, __fmul_rn(static_cast<float>(pw + 1), bin_w))), W);
        const int hs = psroi_edge(floorf(__fadd_rn(y1, __fmul_rn(static_cast<float>(ph), bin_h))), H);
        const int he = psroi_edge(ceilf(__fadd_rn(y1, __fmul_rn(static_cast<float>(ph + 1), bin_h))), H);
        float v = 0.f;
        if (we > ws && he > hs) {
            const int c = (q * PH + ph) * PW + pw;
            const float* plane = in + (static_cast<size_t>(n) * C + c) * H * W;
            float sum = 0.f;
            for (int h = hs; h < he; ++h)
                for (int x = ws; x < we; ++x) sum = __fadd_rn(sum, __ldg(plane + static_cast<size_t>(h) * W + x));
            v = __fdiv_rn(sum, static_cast<float>((he - hs) * (we - ws)));
        }
        out[t] = v;
    }
}

ProposalGeom proposal_geom(const FcudaProposalParam& p, int feat_h, int feat_w) {
    ProposalGeom g{};
    g.A = kProposalAnchors;
    g.H = feat_h;
    g.W = feat_w;
    g.P = kProposalAnchors * feat_h * feat_w;
    g.stride = static_cast<float>(p.feat_stride);
    g.min_size = static_cast<float>(p.min_size);
    float table[kProposalAnchors * 4];
    proposal_anchors(p, table);
    for (int q = 0; q < kProposalAnchors; ++q) {
        g.ax1[q] = table[4 * q];
        g.ay1[q] = table[4 * q + 1];
        g.aw[q] = table[4 * q + 2];
        g.ah[q] = table[4 * q + 3];
    }
    return g;
}

int proposal_decode_launch(float* boxes, uint32_t* keys, int key_stride, const float* score, const float* bbox,
                           const float* im_info, const ProposalGeom& g, int batch, cudaStream_t s) {
    const long long total = static_cast<long long>(batch) * g.P;
    const int prof = prof_begin(s, PROF_RCNN, 0, 0, (keys ? 40.0 : 36.0) * total);
    const long long blocks = (total + 255) / 256;
    proposal_decode_kernel<<<static_cast<unsigned>(blocks < 65536 * 16 ? blocks : 65536 * 16), 256, 0, s>>>(
        reinterpret_cast<float4*>(boxes), keys, key_stride, score, bbox, im_info, g, total);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

SmemAttrCache proposal_select_smem;

}  // namespace

void proposal_anchors(const FcudaProposalParam& p, float* table) {
    const float ratios[3] = {0.5f, 1.f, 2.f}, scales[3] = {8.f, 16.f, 32.f};
    const float base = static_cast<float>(p.base_size);
    for (int r = 0; r < 3; ++r) {
        const float rw = roundf(base / sqrtf(ratios[r]));
        const float rh = roundf(rw * ratios[r]);
        for (int k = 0; k < 3; ++k) {
            const float aw = rw * scales[k], ah = rh * scales[k];
            float* a = table + 4 * (r * 3 + k);
            a[0] = base * 0.5f - aw * 0.5f;
            a[1] = base * 0.5f - ah * 0.5f;
            a[2] = aw;
            a[3] = ah;
        }
    }
}

int proposal_decode(float* boxes, const float* score, const float* bbox, const float* im_info, const FcudaProposalParam& p,
                    int feat_h, int feat_w, int batch, cudaStream_t s) {
    return proposal_decode_launch(boxes, nullptr, 0, score, bbox, im_info, proposal_geom(p, feat_h, feat_w), batch, s);
}

size_t proposal_workspace(const FcudaProposalParam& p, int feat_h, int feat_w, int batch) {
    const size_t P = static_cast<size_t>(kProposalAnchors) * feat_h * feat_w, K = static_cast<size_t>(p.pre_nms_topN);
    const size_t n = static_cast<size_t>(batch);
    return n * (4 * P + round4(P) + 4 * K + 2 * round4(K) + K * ceil_div_sz(K, 32)) + round4(n);
}

int proposal_forward(float* rois, float* scores, const float* score, const float* bbox, const float* im_info,
                     const FcudaProposalParam& p, int feat_h, int feat_w, float* workspace, int batch, cudaStream_t s) {
    const ProposalGeom g = proposal_geom(p, feat_h, feat_w);
    const ProposalWorkspace w = proposal_carve(workspace, g.P, p.pre_nms_topN, batch);
    int rc = proposal_decode_launch(w.boxes, w.keys, w.P4, score, bbox, im_info, g, batch, s);
    if (rc) return rc;
    const double n = batch, K = p.pre_nms_topN;
    int len = 1;
    while (len < p.pre_nms_topN) len <<= 1;
    const int smem = len * static_cast<int>(sizeof(unsigned long long));
    rc = ensure_dynamic_smem(proposal_select_kernel, smem, proposal_select_smem);
    if (rc) return rc;
    int prof = prof_begin(s, PROF_RCNN, 0, 0, n * (4.0 * g.P + 40.0 * K));
    proposal_select_kernel<<<static_cast<unsigned>(batch), kDetThreads, smem, s>>>(w, g.P);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    prof = prof_begin(s, PROF_RCNN, 0, 0, n * (20.0 * K + 2.0 * K * w.words));
    proposal_mask_kernel<<<dim3(static_cast<unsigned>(ceil_div(p.pre_nms_topN, 32)), static_cast<unsigned>(batch)), 256, 0,
                           s>>>(w, p.nms_thresh);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    prof = prof_begin(s, PROF_RCNN, 0, 0, n * p.after_nms_topN * (20.0 + 4.0 * w.words));
    proposal_sweep_kernel<<<static_cast<unsigned>(batch), 32, 0, s>>>(reinterpret_cast<float4*>(rois), scores, score, w,
                                                                      g.A, feat_h * feat_w, p.after_nms_topN);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

int roi_pooling_forward(float* out, const float* in, const float* rois, int C, int H, int W, int R, int pooled_h,
                        int pooled_w, float spatial_scale, int batch, cudaStream_t s) {
    const long long total = static_cast<long long>(batch) * R * C * pooled_h * pooled_w;
    const int prof = prof_begin(s, PROF_RCNN, 0, 0, 4.0 * batch * C * H * W + 16.0 * batch * R + 4.0 * total);
    const long long blocks = (total + 255) / 256;
    roi_pool_kernel<<<static_cast<unsigned>(blocks < 65536 * 16 ? blocks : 65536 * 16), 256, 0, s>>>(
        out, in, rois, C, H, W, R, pooled_h, pooled_w, spatial_scale, total);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

int psroi_pooling_forward(float* out, const float* in, const float* rois, int C, int H, int W, int R, int pooled_h,
                          int pooled_w, int output_dim, float spatial_scale, int batch, cudaStream_t s) {
    const long long total = static_cast<long long>(batch) * R * C;  // C = output_dim * pooled_h * pooled_w
    const int prof = prof_begin(s, PROF_RCNN, 0, 0, 4.0 * batch * C * H * W + 16.0 * batch * R + 4.0 * total);
    const long long blocks = (total + 255) / 256;
    psroi_pool_kernel<<<static_cast<unsigned>(blocks < 65536 * 16 ? blocks : 65536 * 16), 256, 0, s>>>(
        out, in, rois, C, H, W, R, pooled_h, pooled_w, output_dim, spatial_scale, total);
    FCUDA_CHECK_LAUNCH();
    prof_end(prof, s);
    count_launch();
    return 0;
}

}  // namespace fcuda
