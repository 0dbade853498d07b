// Stand-alone self test for the wgmma TensorGEMM kernel (needs an H100).
//   build: make -C feathercnn_b200/csrc selftest      run: build/gemm_selftest [--bench]
// Compares tensor_gemm (TF32 and 3xTF32) against a double-precision host GEMM on small shapes and
// against the CUDA-core fp32 kernel on large ones, for every epilogue.  Exit code != 0 on mismatch.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "../../feathercnn_b200/csrc/tensor_gemm.cuh"

using namespace fcuda;

#define CK(x)                                                                              \
    do {                                                                                   \
        cudaError_t e = (x);                                                               \
        if (e != cudaSuccess) {                                                            \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
            exit(2);                                                                       \
        }                                                                                  \
    } while (0)

static void split_host(const std::vector<float>& v, std::vector<float>& hi, std::vector<float>& lo) {
    hi.resize(v.size());
    lo.resize(v.size());
    for (size_t i = 0; i < v.size(); ++i) {
        uint32_t u;
        memcpy(&u, &v[i], 4);
        uint32_t r = (u + 0x1000u) & 0xFFFFE000u;
        float h;
        memcpy(&h, &r, 4);
        hi[i] = h;
        lo[i] = v[i] - h;
    }
}

struct Case {
    int M, N, K, G, epi, P, split_k;
    bool host_ref;
};

static int run_case(const Case& c, int planes, bool bench) {
    const size_t nA = (size_t)c.G * c.M * c.K, nB = (size_t)c.G * c.N * c.K;
    size_t nD;
    int ldd = 0;
    if (c.epi == EPI_ROWMAJOR) { ldd = c.N; nD = (size_t)c.G * c.M * c.N; }
    else if (c.epi == EPI_NCHW) { nD = (size_t)c.M * c.N; }
    else { ldd = c.M; nD = (size_t)c.N * c.M; }
    std::mt19937 rng(1234 + c.M * 7 + c.N * 13 + c.K);
    std::uniform_real_distribution<float> dist(-1.f, 1.f);
    std::vector<float> A(nA), B(nB), bias(c.N), Ahi, Alo, Bhi, Blo;
    for (auto& x : A) x = dist(rng);
    for (auto& x : B) x = dist(rng);
    for (auto& x : bias) x = dist(rng);
    split_host(A, Ahi, Alo);
    split_host(B, Bhi, Blo);

    float *dAh, *dAl, *dBh, *dBl, *dD, *dR, *dbias;
    CK(cudaMalloc(&dAh, nA * 4)); CK(cudaMalloc(&dAl, nA * 4));
    CK(cudaMalloc(&dBh, nB * 4)); CK(cudaMalloc(&dBl, nB * 4));
    const int splits = c.epi == EPI_COLMAJOR_PARTIAL ? tensor_gemm_effective_split(c.K, c.split_k) : 1;
    CK(cudaMalloc(&dD, nD * 4 * splits)); CK(cudaMalloc(&dR, nD * 4)); CK(cudaMalloc(&dbias, c.N * 4));
    CK(cudaMemcpy(dAh, Ahi.data(), nA * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dAl, Alo.data(), nA * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dBh, Bhi.data(), nB * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dBl, Blo.data(), nB * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dbias, bias.data(), c.N * 4, cudaMemcpyHostToDevice));
    CK(cudaMemset(dD, 0, nD * 4 * splits));
    CK(cudaMemset(dR, 0, nD * 4));

    GemmProblem p{};
    CK(cudaMemcpy(dAh, A.data(), nA * 4, cudaMemcpyHostToDevice));  // A goes in as plain fp32
    p.A = dAh; p.B_hi = dBh; p.B_lo = dBl; p.D = dD;
    p.M = c.M; p.N = c.N; p.K = c.K; p.G = c.G; p.planes = planes; p.epilogue = c.epi; p.ldd = ldd;
    p.P = c.P;
    if (c.epi == EPI_NCHW) p.epi = conv_epilogue(/*activation=*/1, true, dbias, 0.f, 0.f, nullptr, 0, 0);  // bias + ReLU
    p.split_k = c.split_k;
    p.split_stride = (long long)nD;
    int rc = tensor_gemm(p, 0);
    if (rc) { printf("tensor_gemm rc=%d\n", rc); return 1; }
    CK(cudaDeviceSynchronize());

    // reference: fp32 CUDA-core GEMM on hi+lo (== original fp32 values)
    GemmProblem rp = p;
    rp.D = dR; rp.planes = 2; rp.split_k = 1;
    rc = simt_gemm(rp, 0);
    if (rc) { printf("simt_gemm rc=%d\n", rc); return 1; }
    CK(cudaDeviceSynchronize());

    std::vector<float> D(nD), R(nD), parts(nD * splits);
    CK(cudaMemcpy(parts.data(), dD, nD * 4 * splits, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < nD; ++i) {  // fixed-order sum of the k-split planes (what fc_reduce does on the device)
        float v = 0.f;
        for (int sp = 0; sp < splits; ++sp) v += parts[(size_t)sp * nD + i];
        D[i] = v;
    }
    CK(cudaMemcpy(R.data(), dR, nD * 4, cudaMemcpyDeviceToHost));

    double max_ref = 0, max_err = 0, max_err_host = -1;
    for (size_t i = 0; i < nD; ++i) {
        max_ref = fmax(max_ref, fabs((double)R[i]));
        max_err = fmax(max_err, fabs((double)D[i] - (double)R[i]));
    }
    if (c.host_ref) {
        max_err_host = 0;
        for (int g = 0; g < c.G; ++g)
            for (int m = 0; m < c.M; ++m)
                for (int n = 0; n < c.N; ++n) {
                    double s = 0;
                    for (int k = 0; k < c.K; ++k)
                        s += (double)A[((size_t)g * c.M + m) * c.K + k] * (double)B[((size_t)g * c.N + n) * c.K + k];
                    double got;
                    if (c.epi == EPI_ROWMAJOR) got = D[((size_t)g * c.M + m) * ldd + n];
                    else if (c.epi == EPI_NCHW) {
                        s += bias[n];
                        s = s > 0 ? s : 0;
                        int img = m / c.P, pix = m % c.P;
                        got = D[((size_t)img * c.N + n) * c.P + pix];
                    } else got = D[(size_t)n * ldd + m];
                    max_err_host = fmax(max_err_host, fabs(got - s));
                }
    }
    const double rel = max_err / (max_ref > 0 ? max_ref : 1);
    const double tol = planes == 2 ? 5e-5 : 4e-3;  // 3xTF32: fp32-level, summation order differs from the SIMT reference
    const bool ok = rel < tol && (max_err_host < 0 || max_err_host / (max_ref > 0 ? max_ref : 1) < tol);
    printf("M=%6d N=%4d K=%5d G=%3d epi=%d splitk=%d planes=%d : max|ref|=%.3g rel_err_vs_simt=%.3g host_abs_err=%.3g %s\n",
           c.M, c.N, c.K, c.G, c.epi, c.split_k, planes, max_ref, rel, max_err_host, ok ? "OK" : "FAIL");

    if (bench && ok) {
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        for (int i = 0; i < 3; ++i) tensor_gemm(p, 0);
        CK(cudaEventRecord(e0));
        const int iters = 10;
        for (int i = 0; i < iters; ++i) tensor_gemm(p, 0);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        ms /= iters;
        const double flops = 2.0 * c.G * c.M * (double)c.N * c.K;
        const double mma_flops = flops * (planes == 2 ? 3 : 1);
        printf("    time %.3f ms  algorithmic %.1f TFLOP/s  tensor-pipe (incl. 3x) %.1f TFLOP/s\n", ms, flops / ms * 1e-9,
               mma_flops / ms * 1e-9);
    }
    cudaFree(dAh); cudaFree(dAl); cudaFree(dBh); cudaFree(dBl); cudaFree(dD); cudaFree(dR); cudaFree(dbias);
    return ok ? 0 : 1;
}

int main(int argc, char** argv) {
    bool bench = argc > 1 && !strcmp(argv[1], "--bench");
    std::vector<Case> cases = {
        // small, host-checked
        {128, 32, 32, 1, EPI_ROWMAJOR, 1, 1, true},
        {128, 64, 64, 1, EPI_ROWMAJOR, 1, 1, true},
        {100, 24, 36, 2, EPI_ROWMAJOR, 1, 1, true},     // M/N/K tails
        {300, 72, 100, 3, EPI_ROWMAJOR, 1, 1, true},
        {256, 128, 128, 2, EPI_ROWMAJOR, 1, 1, true},
        {200, 160, 64, 1, EPI_ROWMAJOR, 1, 1, true},    // N > 128
        {392, 64, 28, 1, EPI_NCHW, 196, 1, true},       // conv-like: 2 images of 14x14
        {500, 100, 148, 1, EPI_NCHW, 250, 1, true},
        {256, 8, 512, 1, EPI_COLMAJOR_PARTIAL, 1, 1, true},   // FC: M=out, N=batch
        {384, 16, 1024, 1, EPI_COLMAJOR_PARTIAL, 1, 4, true}, // split-K partial planes
        // larger, SIMT-checked
        {6400, 64, 64, 64, EPI_ROWMAJOR, 1, 1, false},       // Winograd conv 64->64 @56x56, batch 64 rows /64
        {1152, 512, 512, 16, EPI_ROWMAJOR, 1, 1, false},
        {12544, 256, 64, 1, EPI_NCHW, 3136, 1, false},        // 1x1 conv 64->256 @56x56, 4 images
        {4096, 64, 25088, 1, EPI_COLMAJOR_PARTIAL, 1, 8, false},  // VGG fc6 @ batch 64
    };
    int fails = 0;
    for (const auto& c : cases)
        for (int planes = 1; planes <= 2; ++planes) fails += run_case(c, planes, bench);
    if (bench) {
        std::vector<Case> perf = {
            {65536, 64, 64, 64, EPI_ROWMAJOR, 1, 1, false},
            {16384, 128, 128, 64, EPI_ROWMAJOR, 1, 1, false},
            {8192, 256, 256, 64, EPI_ROWMAJOR, 1, 1, false},
            {2048, 512, 512, 64, EPI_ROWMAJOR, 1, 1, false},
        };
        for (const auto& c : perf)
            for (int planes = 1; planes <= 2; ++planes) fails += run_case(c, planes, true);
    }
    printf(fails ? "SELFTEST FAILED (%d)\n" : "SELFTEST PASSED\n", fails);
    return fails ? 1 : 0;
}
