// TEST INFRASTRUCTURE (INTEGRATION.md §1, compiled): the file a FeatherCNN maintainer adds to the REFERENCE tree as
// src/booster/cuda/booster.cpp.  It implements the reference's own plugin boundary —
//     booster::ConvBooster::{SelectAlgo, ForceSelectAlgo, SetFuncs} and the GET_BUFFER_SIZE_FUNC / INIT_FUNC /
//     FORWARD_FUNC table     (/root/reference/src/booster/include/booster/booster.h:151-170)
// — on top of the C ABI of libfcuda.so (include/fcuda.h), in place of src/booster/avx/booster.cpp.  oracle/Makefile links
// it with the UNMODIFIED reference objects (feather::Net, ConvLayer, ncnn loader, the AVX element-wise kernels) into
// oracle/_ref/libfeather_ref_cuda.so, and tests/test_gpu_integration.py runs the reference's feather::Net on the GPU
// kernels against the reference's AVX build.  Nothing in the product path includes or links this file.
//
// The reference host keeps HOST blobs and is batch-1 (src/blob.cpp:73), so this binding stages through device memory
// inside Forward; all device buffers are created once in Init (ConvLayer::Init runs after the shapes are known,
// src/layers/conv_layer.h:153-172) and live behind the `processed_kernel` floats the layer owns.
#include <booster/booster.h>

#include <cuda_runtime.h>
#include <fcuda.h>
#include <stdio.h>
#include <string.h>

namespace booster {

static_assert(sizeof(ConvParam) == sizeof(FcudaConvParam), "booster::ConvParam layout drifted from FcudaConvParam");
static inline FcudaConvParam* P(ConvParam* p) { return reinterpret_cast<FcudaConvParam*>(p); }

namespace {

struct DeviceSide {       // stored in the layer's processed_kernel buffer
    float* packed;        // transformed / packed filters
    float* scratch;       // Winograd V / M, im2col rows
    float* in;            // one image
    float* out;
    float* bias;          // OC floats (uploaded at the first Forward: Init does not see the bias, booster.h:152)
    int bias_uploaded;
};
constexpr int kDeviceSideFloats = (sizeof(DeviceSide) + sizeof(float) - 1) / sizeof(float);

#define CU_TRY(expr)                                                                         \
    do {                                                                                     \
        cudaError_t e_ = (expr);                                                             \
        if (e_ != cudaSuccess) {                                                             \
            fprintf(stderr, "cuda booster: %s: %s\n", #expr, cudaGetErrorString(e_));        \
            return -1;                                                                       \
        }                                                                                    \
    } while (0)

size_t in_floats(const ConvParam* p) { return static_cast<size_t>(p->input_channels) * p->input_h * p->input_w; }
size_t out_floats(const ConvParam* p) { return static_cast<size_t>(p->output_channels) * p->output_h * p->output_w; }

// GET_BUFFER_SIZE_FUNC (booster.h:151), sizes in floats (conv_layer.h:112,159).  The host scratch pool is not used by the
// GPU path; the "processed kernel" the layer allocates only has to hold the DeviceSide record.
template <int ALGO>
int CUDA_GetBufferSize(ConvParam* param, int* buffer_size, int* processed_kernel_size) {
    size_t scratch = 0, packed = 0;
    const int rc = fcuda_conv_get_buffer_size(P(param), ALGO, 1, &scratch, &packed);
    if (rc) return rc;
    *buffer_size = 0;
    *processed_kernel_size = kDeviceSideFloats;
    return 0;
}

// INIT_FUNC (booster.h:152): raw host kernel -> transformed device kernel; every device buffer is created here, once.
template <int ALGO>
int CUDA_Init(ConvParam* param, float* processed_kernel, float* kernel) {
    size_t scratch = 0, packed = 0;
    int rc = fcuda_conv_get_buffer_size(P(param), ALGO, 1, &scratch, &packed);
    if (rc) return rc;
    DeviceSide d;
    memset(&d, 0, sizeof(d));
    CU_TRY(cudaMalloc(reinterpret_cast<void**>(&d.packed), (packed ? packed : 1) * sizeof(float)));
    CU_TRY(cudaMalloc(reinterpret_cast<void**>(&d.scratch), (scratch ? scratch : 1) * sizeof(float)));
    CU_TRY(cudaMalloc(reinterpret_cast<void**>(&d.in), in_floats(param) * sizeof(float)));
    CU_TRY(cudaMalloc(reinterpret_cast<void**>(&d.out), out_floats(param) * sizeof(float)));
    CU_TRY(cudaMalloc(reinterpret_cast<void**>(&d.bias), static_cast<size_t>(param->output_channels) * sizeof(float)));
    rc = fcuda_conv_init(P(param), ALGO, d.packed, kernel /* a host pointer is accepted */, nullptr);
    if (rc) return rc;
    CU_TRY(cudaDeviceSynchronize());
    memcpy(processed_kernel, &d, sizeof(d));
    return 0;
}

// FORWARD_FUNC (booster.h:153): host in / out like the AVX backend: H2D, kernels, D2H.
template <int ALGO>
int CUDA_Forward(ConvParam* param, float* output, float* input, float* processed_kernel, float* /*buffer*/, float* bias_arr,
                 int /*num_threads*/) {
    DeviceSide d;
    memcpy(&d, processed_kernel, sizeof(d));
    if (!d.packed) return -1;
    CU_TRY(cudaMemcpyAsync(d.in, input, in_floats(param) * sizeof(float), cudaMemcpyHostToDevice, nullptr));
    if (param->bias_term && bias_arr && !d.bias_uploaded) {
        CU_TRY(cudaMemcpyAsync(d.bias, bias_arr, static_cast<size_t>(param->output_channels) * sizeof(float),
                               cudaMemcpyHostToDevice, nullptr));
        d.bias_uploaded = 1;
        memcpy(processed_kernel, &d, sizeof(d));
    }
    const int rc = fcuda_conv_forward(P(param), ALGO, d.out, d.in, d.packed, d.scratch, param->bias_term ? d.bias : nullptr, 1,
                                      nullptr);
    if (rc) return rc;
    CU_TRY(cudaMemcpyAsync(output, d.out, out_floats(param) * sizeof(float), cudaMemcpyDeviceToHost, nullptr));
    CU_TRY(cudaStreamSynchronize(nullptr));
    return 0;
}

}  // namespace

// ---- the class the reference declares (booster.h:156-170), defined here instead of avx/booster.cpp:283-355 ----
ConvBooster::ConvBooster() : GetBufferSize(NULL), Init(NULL), Forward(NULL) {}

int ConvBooster::SelectAlgo(ConvParam* param) {
    int a = -1;
    const int rc = fcuda_conv_select_algo(P(param), &a);  // the reference's own rule (avx/booster.cpp:283-310)
    if (rc) return rc;
    this->algo = static_cast<ConvAlgo>(a);
    return this->SetFuncs();
}

int ConvBooster::ForceSelectAlgo(ConvAlgo algo) {
    this->algo = algo;
    return this->SetFuncs();
}

#define BIND(A)                                  \
    case A:                                      \
        this->GetBufferSize = CUDA_GetBufferSize<A>; \
        this->Init = CUDA_Init<A>;               \
        this->Forward = CUDA_Forward<A>;         \
        return 0;

int ConvBooster::SetFuncs() {
    switch (this->algo) {
        BIND(NAIVE)
        BIND(IM2COL)
        BIND(SGECONV)
        BIND(DEPTHWISE)
        BIND(WINOGRADF63)
        BIND(WINOGRADF23)
        default:
            fprintf(stderr, "This algo is not supported on the CUDA booster.\n");  // avx/booster.cpp:349-353
            this->GetBufferSize = NULL;
            this->Init = NULL;
            this->Forward = NULL;
            return -1;
    }
}

}  // namespace booster
