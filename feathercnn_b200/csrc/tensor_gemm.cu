// TensorGEMM on Hopper warpgroup MMA (sm_90a).  See tensor_gemm.cuh for the contract.
//
// tensor_gemm_kernel<BN, PLANES, CLIP>: persistent CTAs of 288 threads walk the 128 x BN output tiles (and k-splits) with
// a static stride:
//   warp 8        TMA producer : per 32-wide k-block the raw fp32 A tile (128 rows) and the B_hi (+ B_lo) tiles
//                                (cp.async.bulk.tensor 3-D boxes, 128-byte swizzle) into a kStages-deep smem ring.  It
//                                keeps a running k-block count across tiles, so it fills the next tile's stages while
//                                the consumers run the epilogue.
//   warps 0..7    two consumer warpgroups, 64 rows each: a thread reads its A fragment from the swizzled tile, splits it
//                 into TF32 hi + fp32 lo (PLANES == 2) in registers and issues wgmma.mma_async with A from registers and B
//                 from shared memory: A_lo*B_hi + A_hi*B_lo + A_hi*B_hi per k-step of 8 into fp32 register
//                 accumulators; then the fused store (row-major / NCHW+bias+ReLU / k-split partial planes).
// A is ONE fp32 plane in HBM (the split happens on chip); full / empty mbarriers hand the ring slots over, and a bounded
// wait traps instead of hanging the GPU.
#include "tensor_gemm.cuh"
#include "common.cuh"
#include "wgmma.cuh"

#include <atomic>
#include <string.h>
#include <stdlib.h>
#include <mutex>
#include <vector>

namespace fcuda {

// --------------------------------------------------------------------------------------------
// Kernel
// --------------------------------------------------------------------------------------------
constexpr int kBM = 128;
constexpr int kBK = 32;  // fp32 elements per k-block = 128 bytes = one swizzle atom
constexpr int kConsumerWarps = 8;
constexpr int kThreads = (kConsumerWarps + 1) * 32;
constexpr int kStages = 4;

struct GemmKernelArgs {
    float* D;
    const float* bias;
    int M, N, K, G;
    int epilogue, ldd, P, act, split_k;
    float lo, hi;  // EPI_NCHW, act != 0: the Clip bounds ([0, +inf] for a ReLU, which the simt kernel clamps to)
    int num_m, num_n, k_blocks_total;
    long long m_offset;
    long long split_stride;
    int vec2;  // EPI_ROWMAJOR: pairs of columns leave as one 8-byte store (ldd even, D 8-byte aligned)
};

// Stores the two rows (m0, m0 + 8) x BN/4 column pairs this thread holds through the fused store of args.epilogue.
template <int BN, bool CLIP>
__device__ __forceinline__ void epilogue_store(const GemmKernelArgs& args, const float (&acc)[BN / 2], int g, int m0,
                                               int n_base, int c, int ks) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + 8 * h;
        if (m >= args.M) continue;
        if (args.epilogue == EPI_ROWMAJOR) {
            float* row = args.D + (static_cast<size_t>(g) * args.M + m) * args.ldd;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = n_base + 8 * j + 2 * c;
                const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                if (args.vec2 && n + 1 < args.N) {
                    *reinterpret_cast<float2*>(row + n) = make_float2(v0, v1);
                } else {
                    if (n < args.N) row[n] = v0;
                    if (n + 1 < args.N) row[n + 1] = v1;
                }
            }
        } else if (args.epilogue == EPI_NCHW) {
            const long long mg = args.m_offset + m;
            const int img = static_cast<int>(mg / args.P);
            const int pix = static_cast<int>(mg - static_cast<long long>(img) * args.P);
            float* dst = args.D + static_cast<size_t>(img) * args.N * args.P + pix;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = n_base + 8 * j + 2 * c + e;
                    if (n < args.N) {
                        float v = acc[4 * j + 2 * h + e];
                        if (args.bias) v += __ldg(args.bias + n);
                        if (args.act) v = act_clamp<CLIP>(v, args.lo, args.hi);
                        dst[static_cast<size_t>(n) * args.P] = v;
                    }
                }
            }
        } else {  // EPI_COLMAJOR_PARTIAL: this k-split's plane, plain stores
            float* dst = args.D + static_cast<size_t>(ks) * args.split_stride + m;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = n_base + 8 * j + 2 * c + e;
                    if (n < args.N) dst[static_cast<size_t>(n) * args.ldd] = acc[4 * j + 2 * h + e];
                }
            }
        }
    }
}

// tile = ((ks * G + g) * num_m + m_blk) * num_n + n_blk: neighbouring CTAs share the A tile
struct TileCoord { int g, m_blk, n_blk, ks, kb0, nk; };

__device__ __forceinline__ TileCoord tile_coord(const GemmKernelArgs& args, int tile) {
    TileCoord t;
    t.n_blk = tile % args.num_n;
    const int t1 = tile / args.num_n;
    t.m_blk = t1 % args.num_m;
    const int t2 = t1 / args.num_m;
    t.g = t2 % args.G;
    t.ks = t2 / args.G;
    const int kb_per_split = (args.k_blocks_total + args.split_k - 1) / args.split_k;
    t.kb0 = t.ks * kb_per_split;
    t.nk = min(t.kb0 + kb_per_split, args.k_blocks_total) - t.kb0;
    return t;
}

// This thread's A fragments of one k-block, read from the raw fp32 tile at a_base (128-byte rows, 128-byte swizzle) and
// split as split_fragments does: rows row0 and row0 + 8, whose swizzle phase row & 7 is gq for both.
template <int PLANES>
__device__ __forceinline__ void load_a_fragments(uint32_t a_base, int row0, int gq, int c, uint32_t (&f1)[4][4],
                                                 uint32_t (&f2)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {  // q: a0 (row0, k), a1 (row0 + 8, k), a2 (row0, k + 4), a3 (row0 + 8, k + 4)
            const int row = row0 + 8 * (q & 1);
            const uint32_t chunk = static_cast<uint32_t>(2 * kk + (q >> 1)) ^ static_cast<uint32_t>(gq);
            float x;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(a_base + row * 128 + (chunk << 4) + c * 4));
            if (PLANES == 2) split_tf32_trunc(x, f1[kk][q], f2[kk][q]);
            else f1[kk][q] = __float_as_uint(x);
        }
    }
}

// Two A-fragment sets overlap the k-blocks: k-block kb + 1 is read from the swizzled tile and split while kb's commit
// group runs (wgmma_wait<1>); a ring stage is released once the group that read its B planes retired.
template <int BN, int PLANES, bool CLIP>
__global__ void __launch_bounds__(kThreads, 1)
tensor_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmBlo, const GemmKernelArgs args, int tiles) {
    constexpr int kATile = kBM * kBK * 4;
    constexpr int kBTile = BN * kBK * 4;
    constexpr int kStage = kATile + PLANES * kBTile;  // [A raw][B_hi][B_lo]
    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment.
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ uint64_t full_bar[kStages];
    __shared__ uint64_t empty_bar[kStages];

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        ptx::mbar_init_ring(full_bar, empty_bar, kStages, kConsumerWarps);
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            ptx::prefetch_tensormap(&tmA);
            ptx::prefetch_tensormap(&tmB);
            if (PLANES == 2) ptx::prefetch_tensormap(&tmBlo);
            int kbg = 0;  // k-blocks issued by this CTA over all its tiles
            for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                const TileCoord tc = tile_coord(args, tile);
                for (int i = 0; i < tc.nk; ++i, ++kbg) {
                    const int stage = kbg % kStages;
                    if (kbg >= kStages) ptx::mbar_wait(&empty_bar[stage], ((kbg / kStages) - 1) & 1);
                    uint8_t* st = smem + stage * kStage;
                    const int kc = (tc.kb0 + i) * kBK;
                    ptx::mbar_arrive_expect_tx(&full_bar[stage], kStage);
                    ptx::tma_load_3d(st, &tmA, &full_bar[stage], kc, tc.m_blk * kBM, tc.g);
                    ptx::tma_load_3d(st + kATile, &tmB, &full_bar[stage], kc, tc.n_blk * BN, tc.g);
                    if (PLANES == 2) ptx::tma_load_3d(st + kATile + kBTile, &tmBlo, &full_bar[stage], kc, tc.n_blk * BN, tc.g);
                }
            }
        }
        return;
    }

    // ===================== consumers: two warpgroups of 64 rows =====================
    const int gq = lane >> 2, c = lane & 3;
    const int row0 = warp * 16 + gq;
    int kbg = 0;  // k-blocks consumed by this CTA over all its tiles
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const TileCoord tc = tile_coord(args, tile);
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        uint32_t fa1[4][4], fa2[4][4], fb1[4][4], fb2[4][4];  // two fragment sets: [k-step][a0..a3], hi and lo

        auto step = [&](uint32_t (&f1)[4][4], uint32_t (&f2)[4][4], int i) {
            const int stage = kbg % kStages;
            ptx::mbar_wait(&full_bar[stage], (kbg / kStages) & 1);
            const uint32_t a_base = ptx::smem_u32(smem + stage * kStage);
            load_a_fragments<PLANES>(a_base, row0, gq, c, f1, f2);
            ptx::wgmma_fence();
            mma_kblock<BN, PLANES>(acc, f1, f2, a_base + kATile, a_base + kATile + kBTile);
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();  // k-block i - 1 retired: its stage's B planes and its fragment set are free
            __syncwarp();
            ptx::mbar_arrive_if(&empty_bar[(kbg + kStages - 1) % kStages], i > 0 && lane == 0);
            ++kbg;
        };
        // k-blocks in pairs, one per fragment set.  Both loop shapes issue the same sequence; ptxas keeps the wgmma
        // pipelined only with the odd tail inside the loop for PLANES 2 (else C7512) and after it for PLANES 1 (else C7513).
        if (PLANES == 2) {
            for (int i = 0; i < tc.nk; i += 2) {
                step(fa1, fa2, i);
                if (i + 1 < tc.nk) step(fb1, fb2, i + 1);
            }
        } else {
            int i = 0;
            for (; i + 1 < tc.nk; i += 2) {
                step(fa1, fa2, i);
                step(fb1, fb2, i + 1);
            }
            if (i < tc.nk) step(fa1, fa2, i);
        }
        ptx::wgmma_wait<0>();
        __syncwarp();
        ptx::mbar_arrive_if(&empty_bar[(kbg - 1) % kStages], lane == 0);  // the producer refills it during the epilogue
        epilogue_store<BN, CLIP>(args, acc, tc.g, tc.m_blk * kBM + row0, tc.n_blk * BN, c, tc.ks);
    }
}

// --------------------------------------------------------------------------------------------
// Host side
// --------------------------------------------------------------------------------------------
EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        // Resolve through the runtime so the library does not link libcuda directly.
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

static std::atomic<unsigned long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(static_cast<unsigned long long>(n), std::memory_order_relaxed); }
unsigned long long launch_count() { return g_launches.load(std::memory_order_relaxed); }
void reset_launch_count() { g_launches.store(0, std::memory_order_relaxed); }

// ---- kernel-variant switches ---------------------------------------------------------------------------------------
namespace {
struct TuneEntry { const char* name; const char* env; int def, lo, hi; int value; bool init; };
TuneEntry g_tune[TUNE_COUNT] = {
    {"dw_vec", "FCUDA_DW_VEC", 1, 0, 1, 0, false},                   // vectorised depthwise kernel on wide planes
    {"igemm_halo", "FCUDA_IGEMM_HALO", 1, 0, 1, 0, false},           // implicit GEMM: TMA halo tiles + pipelined wgmma (stride 1)
    {"igemm_presplit", "FCUDA_IGEMM_PRESPLIT", 1, 0, 1, 0, false},   // BF16x3 halo kernel: one split per box, ldmatrix fragments
    {"igemm_wide", "FCUDA_IGEMM_WIDE", 1, 0, 1, 0, false},           // pre-split kernel: 224-pixel N side, filters on M
    {"igemm_stem", "FCUDA_IGEMM_STEM", 1, 0, 1, 0, false},           // short-K k-table layers: persistent, resident filters
    {"route_fuse", "FCUDA_ROUTE_FUSE", 1, 0, 1, 0, false},           // Net fusion: Concat -> ShuffleChannel -> Slice in one launch
    {"persistent_ctas", "FCUDA_PERSISTENT_CTAS", 0, 0, 65536, 0, false},  // n > 0: persistent kernels run at most n CTAs
};
}  // namespace
const char* tune_name(int key) { return key >= 0 && key < TUNE_COUNT ? g_tune[key].name : nullptr; }
int tune_get(int key) {
    if (key < 0 || key >= TUNE_COUNT) return 0;
    TuneEntry& e = g_tune[key];
    if (!e.init) {
        e.value = e.def;
        if (const char* v = getenv(e.env)) {
            const int x = atoi(v);
            if (x >= e.lo && x <= e.hi) e.value = x;
        }
        e.init = true;
    }
    return e.value;
}
int tune_set(const char* name, int value) {
    if (!name) return -200;
    for (int k = 0; k < TUNE_COUNT; ++k)
        if (!strcmp(name, g_tune[k].name)) {
            if (value < g_tune[k].lo || value > g_tune[k].hi || false) return -200;
            g_tune[k].value = value;
            g_tune[k].init = true;
            return 0;
        }
    return -200;
}

// ---- per-launch profiling ------------------------------------------------------------------------
// Off by default.  When enabled every instrumented launch is bracketed by two CUDA events on its own stream and tagged
// with its kernel class and ALGORITHMIC work (the FLOPs / bytes the operation needs, not what the kernel happens to
// move), which is what bench.py divides by the measured time for the roofline object.
struct ProfRec { cudaEvent_t e0, e1; int kind; double algo_flops, mma_flops, algo_bytes; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;

void gemm_profile_enable(bool on) {
    if (on) {
        for (auto& r : g_prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
        g_prof.clear();
    }
    g_prof_on = on;
}

int prof_begin(cudaStream_t s, int kind, double algo_flops, double mma_flops, double algo_bytes) {
    if (!g_prof_on) return -1;
    ProfRec rec{};
    rec.kind = kind; rec.algo_flops = algo_flops; rec.mma_flops = mma_flops; rec.algo_bytes = algo_bytes;
    cudaEventCreate(&rec.e0);
    cudaEventCreate(&rec.e1);
    cudaEventRecord(rec.e0, s);
    g_prof.push_back(rec);
    return static_cast<int>(g_prof.size()) - 1;
}
void prof_end(int idx, cudaStream_t s) {
    if (idx >= 0 && idx < static_cast<int>(g_prof.size())) cudaEventRecord(g_prof[idx].e1, s);
}

// kind < 0: all classes
void profile_collect_kind(int kind, double* total_ms, double* algo_flops, double* mma_flops, double* algo_bytes,
                          long long* launches) {
    double ms = 0, af = 0, mf = 0, ab = 0;
    long long n = 0;
    for (auto& r : g_prof) {
        if (kind >= 0 && r.kind != kind) continue;
        float t = 0.f;
        if (cudaEventSynchronize(r.e1) == cudaSuccess && cudaEventElapsedTime(&t, r.e0, r.e1) == cudaSuccess) ms += t;
        af += r.algo_flops; mf += r.mma_flops; ab += r.algo_bytes; ++n;
    }
    if (total_ms) *total_ms = ms;
    if (algo_flops) *algo_flops = af;
    if (mma_flops) *mma_flops = mf;
    if (algo_bytes) *algo_bytes = ab;
    if (launches) *launches = n;
}
void gemm_profile_collect(double* total_ms, double* algo_flops, double* mma_flops, long long* launches) {
    profile_collect_kind(PROF_TENSOR_GEMM, total_ms, algo_flops, mma_flops, nullptr, launches);
}

// A read once + B read once + D written once (fp32), the least a GEMM of these shapes must move
static double gemm_algo_bytes(const GemmProblem& p) {
    return 4.0 * p.G * (static_cast<double>(p.M) * p.K + static_cast<double>(p.N) * p.K * (p.planes == 2 ? 2 : 1) +
                        static_cast<double>(p.M) * p.N);
}

int sm_count() {
    static int n[kMaxDevices] = {};
    const int dev = current_device();
    if (n[dev] == 0) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) return 132;
        n[dev] = v;
    }
    return n[dev];
}

int make_map(CUtensorMap* map, const float* base, int K, int rows, int G, long long batch_stride, int box_rows) {
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) {
        fprintf(stderr, "fcuda: cuTensorMapEncodeTiled unavailable (no CUDA driver?)\n");
        return FCUDA_ERR_CUDA;
    }
    cuuint64_t dims[3] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(G)};
    const cuuint64_t bstride = batch_stride > 0 ? static_cast<cuuint64_t>(batch_stride)
                                                : static_cast<cuuint64_t>(K) * static_cast<cuuint64_t>(rows);
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(K) * 4, bstride * 4};
    cuuint32_t box[3] = {static_cast<cuuint32_t>(kBK), static_cast<cuuint32_t>(box_rows), 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "fcuda: cuTensorMapEncodeTiled failed (%d) K=%d rows=%d G=%d\n", static_cast<int>(r), K, rows, G);
        return FCUDA_ERR_CUDA;
    }
    return 0;
}

bool tensor_gemm_supported(const GemmProblem& p) {
    if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.G <= 0) return false;
    if (p.K % 4 != 0) return false;
    auto aligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if (!aligned(p.A) || !aligned(p.B_hi)) return false;
    if (p.planes == 2 && (!p.B_lo || !aligned(p.B_lo))) return false;
    if (p.a_batch_stride % 4 != 0 || p.b_batch_stride % 4 != 0) return false;
    return true;
}

static void fill_kernel_args(const GemmProblem& p, int bn, GemmKernelArgs* a) {
    a->D = p.D; a->bias = p.epi.bias;
    a->M = p.M; a->N = p.N; a->K = p.K; a->G = p.G;
    a->epilogue = p.epilogue; a->ldd = p.ldd; a->P = p.P > 0 ? p.P : 1;
    a->act = p.epi.act; a->lo = p.epi.lo; a->hi = p.epi.hi;
    a->m_offset = p.m_offset;
    a->split_stride = p.split_stride;
    a->num_m = ceil_div(p.M, kBM);
    a->num_n = ceil_div(p.N, bn);
    a->k_blocks_total = ceil_div(p.K, kBK);
    a->split_k = tensor_gemm_effective_split(p.K, p.split_k);
    a->vec2 = (p.ldd % 2 == 0 && (reinterpret_cast<uintptr_t>(p.D) & 7) == 0) ? 1 : 0;
}

int tensor_gemm_effective_split(int K, int split_k) {
    const int kb = ceil_div(K, kBK);
    int s = split_k > 0 ? split_k : 1;
    if (s > kb) s = kb;
    // every k-split must own at least one k-block, otherwise its partial plane is never written
    while (s > 1 && ceil_div(kb, s) * (s - 1) >= kb) --s;
    return s;
}

template <int BN, int PLANES, bool CLIP>
static int launch(const GemmProblem& p, cudaStream_t stream) {
    constexpr int kStage = kBM * kBK * 4 + PLANES * BN * kBK * 4;
    static_assert(kStages * kStage + 1024 <= 227 * 1024, "smem budget");
    CUtensorMap tmA, tmB, tmBlo;
    const long long as = p.a_batch_stride ? p.a_batch_stride : static_cast<long long>(p.M) * p.K;
    const long long bs = p.b_batch_stride ? p.b_batch_stride : static_cast<long long>(p.N) * p.K;
    int rc;
    if ((rc = make_map(&tmA, p.A, p.K, p.M, p.G, as, kBM))) return rc;
    if ((rc = make_map(&tmB, p.B_hi, p.K, p.N, p.G, bs, BN))) return rc;
    tmBlo = tmB;
    if (PLANES == 2 && (rc = make_map(&tmBlo, p.B_lo, p.K, p.N, p.G, bs, BN))) return rc;
    GemmKernelArgs a;
    fill_kernel_args(p, BN, &a);
    const long long total = static_cast<long long>(a.num_m) * a.num_n * a.G * a.split_k;
    if (total > 0x7fffffffLL) return -1;
    const int smem = kStages * kStage + 1024;
    auto kern = tensor_gemm_kernel<BN, PLANES, CLIP>;
    static SmemAttrCache attr_cache;
    if (int rc2 = ensure_dynamic_smem(kern, smem, attr_cache)) return rc2;
    unsigned grid = 0;
    if (int rc2 = persistent_grid(kern, kThreads, smem, total, &grid)) return rc2;
    const double dense = 2.0 * p.M * static_cast<double>(p.N) * p.K * p.G;
    const int prof = prof_begin(stream, PROF_TENSOR_GEMM, p.algo_flops > 0 ? p.algo_flops : dense,
                                dense * (PLANES == 2 ? 3.0 : 1.0), gemm_algo_bytes(p));
    kern<<<grid, kThreads, smem, stream>>>(tmA, tmB, tmBlo, a, static_cast<int>(total));
    FCUDA_CHECK_LAUNCH();
    count_launch();
    prof_end(prof, stream);
    return 0;
}

// N tile: the smallest supported tile that covers N (fewer wasted MMA columns), capped at 128.  CLIP: the instantiations
// whose EPI_NCHW epilogue clamps to [epi.lo, epi.hi]; the others apply a ReLU as fmaxf(v, 0).
template <bool CLIP>
static int launch_tile(const GemmProblem& p, cudaStream_t stream) {
    if (p.planes == 2) {
        if (p.N <= 32) return launch<32, 2, CLIP>(p, stream);
        if (p.N <= 64) return launch<64, 2, CLIP>(p, stream);
        return launch<128, 2, CLIP>(p, stream);
    }
    if (p.N <= 32) return launch<32, 1, CLIP>(p, stream);
    if (p.N <= 64) return launch<64, 1, CLIP>(p, stream);
    return launch<128, 1, CLIP>(p, stream);
}

int tensor_gemm(const GemmProblem& p, cudaStream_t stream) {
    if (!tensor_gemm_supported(p)) return -1;
    if (p.split_k > 1 && p.epilogue != EPI_COLMAJOR_PARTIAL) return -1;
    return p.epi.act == 2 ? launch_tile<true>(p, stream) : launch_tile<false>(p, stream);
}

// --------------------------------------------------------------------------------------------
// CUDA-core reference GEMM (same contract).  64x64 tile, 4x4 micro-tile per thread.
// --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
simt_gemm_kernel(const float* __restrict__ A_hi, const float* __restrict__ A_lo, const float* __restrict__ B_hi,
                 const float* __restrict__ B_lo, long long a_stride, long long b_stride, GemmKernelArgs args) {
    __shared__ float sA[16][64 + 4];
    __shared__ float sB[16][64 + 4];
    const int g = blockIdx.z;
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    const float* Ah = A_hi + g * a_stride;
    const float* Al = A_lo ? A_lo + g * a_stride : nullptr;
    const float* Bh = B_hi + g * b_stride;
    const float* Bl = B_lo ? B_lo + g * b_stride : nullptr;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < args.K; k0 += 16) {
        for (int i = threadIdx.x; i < 64 * 16; i += 256) {
            const int r = i >> 4, c = i & 15;
            const int k = k0 + c;
            float a = 0.f, b = 0.f;
            if (m0 + r < args.M && k < args.K) {
                a = Ah[static_cast<size_t>(m0 + r) * args.K + k];
                if (Al) a += Al[static_cast<size_t>(m0 + r) * args.K + k];
            }
            if (n0 + r < args.N && k < args.K) {
                b = Bh[static_cast<size_t>(n0 + r) * args.K + k];
                if (Bl) b += Bl[static_cast<size_t>(n0 + r) * args.K + k];
            }
            sA[c][r] = a;
            sB[c][r] = b;
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = sA[c][ty * 4 + i]; b[i] = sB[c][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= args.M) continue;
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= args.N) continue;
            float v = acc[i][j];
            if (args.epilogue == EPI_ROWMAJOR) {
                args.D[(static_cast<size_t>(g) * args.M + m) * args.ldd + n] = v;
            } else if (args.epilogue == EPI_NCHW) {
                const long long mg = args.m_offset + m;
                const int img = static_cast<int>(mg / args.P), pix = static_cast<int>(mg - static_cast<long long>(img) * args.P);
                if (args.bias) v += args.bias[n];
                if (args.act) v = fminf(fmaxf(v, args.lo), args.hi);
                args.D[(static_cast<size_t>(img) * args.N + n) * args.P + pix] = v;
            } else {
                args.D[static_cast<size_t>(n) * args.ldd + m] = v;
            }
        }
    }
}

int simt_gemm(const GemmProblem& p, cudaStream_t stream) {
    GemmKernelArgs a;
    a.D = p.D; a.bias = p.epi.bias;
    a.M = p.M; a.N = p.N; a.K = p.K; a.G = p.G;
    a.epilogue = p.epilogue; a.ldd = p.ldd; a.P = p.P > 0 ? p.P : 1; a.split_k = 1; a.m_offset = p.m_offset; a.split_stride = 0;
    a.num_m = ceil_div(p.M, 64); a.num_n = ceil_div(p.N, 64); a.k_blocks_total = 0;
    a.act = p.epi.act; a.lo = p.epi.lo; a.hi = p.epi.hi;
    const long long as = p.a_batch_stride ? p.a_batch_stride : static_cast<long long>(p.M) * p.K;
    const long long bs = p.b_batch_stride ? p.b_batch_stride : static_cast<long long>(p.N) * p.K;
    dim3 grid(a.num_n, a.num_m, p.G);
    simt_gemm_kernel<<<grid, 256, 0, stream>>>(p.A, nullptr, p.B_hi, p.planes == 2 ? p.B_lo : nullptr, as, bs, a);
    FCUDA_CHECK_LAUNCH();
    return 0;
}

}  // namespace fcuda
