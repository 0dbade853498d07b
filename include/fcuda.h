/* fcuda.h — C ABI of the H100 (sm_90a) compute backend that replaces FeatherCNN's `booster`.
 *
 * Every entry point cites the reference interface it replaces (paths relative to /root/reference).
 * Conventions, all inherited from the reference boundary (SURVEY.md §8b):
 *   - plain pointers and sizes only; all tensor pointers are DEVICE pointers unless a parameter says "host";
 *   - tensors are fp32, NCHW, channel stride exactly H*W (src/blob.cpp:86-93); a leading batch dimension
 *     `batch` (images, image stride C*H*W) is the one extension — the reference is batch-1 (src/blob.cpp:73);
 *   - buffer sizes are in FLOATS, not bytes (src/layers/conv_layer.h:112,159);
 *   - the library allocates nothing on the hot path: the caller owns outputs, packed kernels and scratch
 *     (src/booster/include/booster/booster.h:155);
 *   - return 0 on success, negative int on failure: -1 unsupported algorithm / partial groups
 *     (src/booster/avx/booster.cpp:306-307,349-353), -100 bad sizes, -200 unsupported parameter, -700 CUDA error;
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); calls are asynchronous.
 */
#ifndef FCUDA_H
#define FCUDA_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* booster::ConvAlgo, src/booster/include/booster/booster.h:42-51 (same numbering). */
enum FcudaConvAlgo {
    FCUDA_NAIVE = 0,            /* CUDA-core fp32 implicit GEMM (device-side second opinion) */
    FCUDA_IM2COL = 1,           /* pack kernel + wgmma TensorGEMM, bias/ReLU fused in the epilogue */
    FCUDA_SGECONV = 2,          /* implicit GEMM straight from NCHW: patches gathered inside the wgmma kernel, no packed
                                   intermediate; a stub in the reference's AVX dispatcher (avx/booster.cpp:105-118) */
    FCUDA_DEPTHWISE = 3,        /* warp-shuffle stencil */
    FCUDA_WINOGRADF63 = 4,      /* F(6,3): input transform -> 64-way wgmma TensorGEMM -> output transform(+bias+ReLU) */
    FCUDA_WINOGRADF63FUSED = 5, /* not selected by the reference (avx/booster.cpp:291-292); unsupported (-1) */
    FCUDA_WINOGRADF23 = 6       /* F(2,3): 16-way TensorGEMM; stub in both reference dispatchers, real here */
};

/* booster::ActivationType, booster.h:53-57, plus FCUDA_ACT_CLIP (ncnn's Clip / Caffe's ReLU6, an extension): a clamp to
 * [clip_min, clip_max] whose bounds fcuda_conv_forward_opts and fcuda_conv_forward_clip carry — every other convolution
 * entry point returns -200 for it. */
enum FcudaActivation { FCUDA_ACT_NONE = 0, FCUDA_ACT_RELU = 1, FCUDA_ACT_CLIP = 2 };

/* Field-compatible with booster::ConvParam (booster.h:59-77): 15 ints, bool, enum. */
typedef struct FcudaConvParam {
    int output_channels;
    int input_channels;
    int input_h;
    int input_w;
    int kernel_h;
    int kernel_w;
    int output_h;
    int output_w;
    int stride_h;
    int stride_w;
    int pad_left;
    int pad_bottom;
    int pad_right;
    int pad_top;
    int group;
    unsigned char bias_term; /* bool */
    int activation;          /* FcudaActivation */
} FcudaConvParam;

/* Arithmetic mode of the tensor-core contraction (global, default FCUDA_PRECISION_FP32_SPLIT).  The tensor cores have no
 * fp32 MMA; every mode accumulates in fp32.
 *   FP32_SPLIT: fp32-equivalent results from split operands, the cheapest split per kernel: the implicit GEMM (SGECONV)
 *               uses BF16x3 — x = p1 + p2 + r with p1 = RN_bf16(x), p2 = RN_bf16(x - p1), three bf16 MMAs
 *               p2*q1 + p1*q2 + p1*q1, dropped terms <= 3 * 2^-16 of a product (measured ~1e-5 of max|out| per layer) at
 *               twice the tensor throughput of 3xTF32; the Winograd / im2col / InnerProduct TensorGEMM keeps 3xTF32
 *               (F(6,3) amplifies operand rounding ~40x).
 *   TF32X3    : every contraction as TF32 hi + fp32 lo planes, 3 TF32 MMAs per k-step (~2^-21 per product).
 *   TF32      : single TF32 MMA — ~2.5e-4 relative error per layer, 3x fewer MMAs. */
enum FcudaPrecision { FCUDA_PRECISION_TF32X3 = 0, FCUDA_PRECISION_TF32 = 1, FCUDA_PRECISION_FP32_SPLIT = 2 };
int fcuda_set_precision(int precision);
int fcuda_get_precision(void);

/* Upper bound (bytes) on the Winograd / im2col intermediates of one chunk: a layer whose packed operands exceed it is
 * processed in several pack -> TensorGEMM -> unpack rounds over the batch (default 8 GiB, i.e. one round for the
 * benchmark configs; 0 = never chunk). */
int fcuda_set_l2_chunk_bytes(size_t bytes);
size_t fcuda_get_l2_chunk_bytes(void);

/* ConvParam::AssignOutputDim, booster.h:113-125. */
int fcuda_conv_assign_output_dim(FcudaConvParam* param);

/* ConvBooster::SelectAlgo, avx/booster.cpp:283-310 (same rule, same -1 for partial groups). */
int fcuda_conv_select_algo(const FcudaConvParam* param, int* algo);

/* Tuned cost-model variant of SelectAlgo: starts from the reference rule and moves bandwidth-bound Winograd layers
 * (<= 128 channels on images >= 28 wide) and the im2col layers to FCUDA_SGECONV.  Unlike the reference rule it treats
 * group == 1 with one input channel as an ordinary convolution, requires group > 1 and OC == IC for FCUDA_DEPTHWISE, and
 * sends partial groups / channel-multiplier depthwise to the grouped FCUDA_SGECONV instead of returning -1. */
int fcuda_conv_select_algo_tuned(const FcudaConvParam* param, int* algo);

/* GET_BUFFER_SIZE_FUNC, booster.h:151: scratch and processed-kernel sizes in floats for `batch` images. */
int fcuda_conv_get_buffer_size(const FcudaConvParam* param, int algo, int batch, size_t* scratch_floats,
                               size_t* packed_kernel_floats);

/* INIT_FUNC, booster.h:152: transforms/packs the raw (OC, IC/group, KH, KW) kernel once.
 * `raw_kernel` may be a host or a device pointer.  Synchronous with respect to `raw_kernel`. */
int fcuda_conv_init(const FcudaConvParam* param, int algo, float* packed_kernel, const float* raw_kernel,
                    void* stream);

/* FORWARD_FUNC, booster.h:153: output (batch, OC, OH, OW) <- input (batch, IC, H, W).
 * `bias` is OC floats or NULL when !bias_term; param->activation fuses ReLU (conv_layer.h:174-185). */
int fcuda_conv_forward(const FcudaConvParam* param, int algo, float* output, const float* input,
                       const float* packed_kernel, float* scratch, const float* bias, int batch, void* stream);

/* What a convolution does beyond fcuda_conv_forward, which is the all-zero struct.  Per output value, in this order:
 * + bias, param->activation (or, with a residual, + residual then relu_after_add), the pooling.
 *   residual        a tensor shaped like the output, added to conv(input) [+bias]: a fused Eltwise SUM (ResNet shortcuts;
 *                   ConvLayer::Forward then EltwiseLayer::Forward, src/layers/eltwise_layer.h:68-82 -> booster::add_relu<>).
 *                   FCUDA_SGECONV with FCUDA_ACT_NONE adds it in its epilogue; every other case runs the convolution with
 *                   its own activation and then add_relu in place.  NULL = none.
 *   relu_after_add  a ReLU after that sum; read only with a residual.
 *   clip_min/max    the bounds of FCUDA_ACT_CLIP: output = min(max(conv(input) [+bias], clip_min), clip_max), the clamp
 *                   applied in the epilogue of the same kernels every algorithm runs, by their Clip instantiations (Caffe's
 *                   ReLU6 is 0, 6).  The bits before the clamp are those of FCUDA_ACT_NONE.  NaN maps to clip_min (fmaxf
 *                   returns the non-NaN operand); ncnn's compare-and-assign Clip passes NaN through.  -200 for
 *                   clip_min > clip_max or a NaN bound, and for a non-zero bound with any other activation.
 *   dilation_h/w    tap spacing, 0 meaning 1 (the reference rejects it, src/layers/conv_layer.h:43-47).  > 1:
 *                   FCUDA_SGECONV and FCUDA_DEPTHWISE only (-200 otherwise, and -200 with a residual that the algorithm
 *                   cannot add in its epilogue, which FCUDA_DEPTHWISE never does); the caller sets param->output_h/w for the
 *                   dilated extent out = (in + pads - dilation*(k-1) - 1) / stride + 1.  < 0: -100.
 *                   FCUDA_DEPTHWISE with a dilation: a 3x3 / stride-1 layer (DeepLab's atrous backbone, pad = dilation)
 *                   computes each output as v = bias, then the nine taps in row-major order, each v = fmaf(w, x, v) with
 *                   x = 0 outside the image, then the activation's clamp.  Every other kernel size or stride adds the taps
 *                   inside the image in row-major order by fmaf from 0, then the bias, then the clamp.  Either way an
 *                   output depends only on its own window, so the bits do not change with the batch split, the pointers'
 *                   alignment or CUDA-graph replay.  A dilation of 1 runs the undilated depthwise kernels unchanged.
 *   pool            non-zero: a FOLLOWING 2x2 / stride-2 / pad-0 max pooling (ConvLayer::Forward then PoolingLayer::Forward,
 *                   src/layers/pooling_layer.h:38-91): `output` is the pooled blob (batch, OC, (OH+1)/2, (OW+1)/2), ceil
 *                   mode, windows clipped at the border like the reference.  -200 unless fcuda_conv_can_pool.
 * Not built, -200: Clip together with a residual or the pooling, or with a dilation outside FCUDA_DEPTHWISE; the pooling
 * together with a residual or a dilation. */
typedef struct FcudaConvOptions {
    const float* residual;
    int relu_after_add;
    float clip_min, clip_max;
    int dilation_h, dilation_w;
    int pool;
} FcudaConvOptions;
/* fcuda_conv_forward with `options` (NULL = the all-zero struct).  The entry points fcuda_conv_forward_clip, _residual,
 * _pool and _ext below are this call with some of the options set. */
int fcuda_conv_forward_opts(const FcudaConvParam* param, int algo, float* output, const float* input,
                            const float* packed_kernel, float* scratch, const float* bias, const FcudaConvOptions* options,
                            int batch, void* stream);

/* fcuda_conv_forward_opts with only clip_min / clip_max set; -200 unless param->activation == FCUDA_ACT_CLIP. */
int fcuda_conv_forward_clip(const FcudaConvParam* param, int algo, float* output, const float* input,
                            const float* packed_kernel, float* scratch, const float* bias, float clip_min, float clip_max,
                            int batch, void* stream);

/* The 64-way batched "TensorGEMM" itself (avx/winograd_kernels_F63.cpp:518-757), exposed for tests and
 * profiling:  for g < G:  D[g][m][n] = sum_k A[g][m][k] * B[g][n][k]   (row-major, K-major operands).
 * `a` is plain fp32 (split into TF32 hi + fp32 lo inside the kernel, in registers); b_hi/b_lo are the planes of
 * fcuda_split_tf32(b) (b_lo NULL => plain TF32 on a and b_hi). */
int fcuda_tensor_gemm(float* d, const float* a, const float* b_hi, const float* b_lo, int m, int n, int k, int g,
                      void* stream);
/* Elementwise TF32 split used to prepare TensorGEMM operands: hi + lo == x exactly. */
int fcuda_split_tf32(float* hi, float* lo, const float* x, size_t n, void* stream);

/* InnerProductLayer (src/layers/inner_product_layer.h:33-170; sgemv.cpp:317-395): z = W x + b per image. */
int fcuda_inner_product_get_buffer_size(int input_size, int output_size, int batch, size_t* scratch_floats,
                                        size_t* packed_kernel_floats);
int fcuda_inner_product_init(int input_size, int output_size, float* packed_kernel, const float* raw_kernel,
                             void* stream);
int fcuda_inner_product_forward(int input_size, int output_size, float* output, const float* input,
                                const float* packed_kernel, const float* bias, float* scratch, int relu, int batch,
                                void* stream);

/* PoolingLayer::Forward (src/layers/pooling_layer.h:38-91) incl. its ceil-mode output size (:129-130,
 * fcuda_pooling_out_dim) and its window start that subtracts both pads (:56,:67). type 0 = max, else average. */
int fcuda_pooling_out_dim(int in, int pad_a, int pad_b, int kernel, int stride);
int fcuda_pooling_forward(float* output, const float* input, int channels, int in_h, int in_w, int type,
                          int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_left, int pad_right,
                          int pad_top, int pad_bottom, int global_pooling, int batch, void* stream);

/* booster::batchnorm<has_bias,has_scale,has_relu> (avx/generic_kernels.cpp:237-279):
 * y = beta[c]*x + alpha[c]; then *scale[c] (if scale), +scale_bias[c] (if scale_bias), ReLU (if relu). */
int fcuda_batchnorm_forward(float* output, const float* input, int channels, size_t stride, const float* alpha,
                            const float* beta, const float* scale, const float* scale_bias, int relu, int batch,
                            void* stream);
/* booster::scale<has_bias> (avx/generic_kernels.cpp:203-233): y = x*scale[c] (+bias[c]). */
int fcuda_scale_forward(float* output, const float* input, int channels, size_t stride, const float* scale,
                        const float* bias, int batch, void* stream);
/* booster::add_relu<fuse_relu> (avx/generic_kernels.cpp:138-169). */
int fcuda_eltwise_add_forward(float* output, const float* a, const float* b, size_t n, int relu, void* stream);
/* Eltwise operations the reference rejects (src/layers/eltwise_layer.h:57-66), with ncnn's semantics:
 * op 0 PROD a*b, op 1 SUM coeff_a*a + coeff_b*b, op 2 MAX max(a,b); optional ReLU.  In-place (output == a) is allowed. */
int fcuda_eltwise_forward(float* output, const float* a, const float* b, size_t n, int op, float coeff_a, float coeff_b,
                          int relu, void* stream);
/* ncnn's BinaryOp (what onnx2ncnn writes for ONNX Add / Sub / Mul / Div / Max / Min / Pow and pnnx for torch.add, x + y,
 * x * 0.5; the reference has no such layer), in ncnn's op numbering.  All arithmetic is fp32, one operation per element:
 * IEEE division and round-to-nearest add / sub / mul.  MAX and MIN are fmaxf / fminf, so a NaN operand yields the other
 * operand (the NaN rule of the Eltwise MAX); the rest propagate NaN.  POW, RPOW, ATAN2 and RATAN2 are CUDA's powf /
 * atan2f, within the ulp bounds the CUDA C Programming Guide lists for them. */
enum FcudaBinaryOp {
    FCUDA_BINARY_ADD = 0,    /* a + b */
    FCUDA_BINARY_SUB = 1,    /* a - b */
    FCUDA_BINARY_MUL = 2,    /* a * b */
    FCUDA_BINARY_DIV = 3,    /* a / b */
    FCUDA_BINARY_MAX = 4,    /* fmaxf(a, b) */
    FCUDA_BINARY_MIN = 5,    /* fminf(a, b) */
    FCUDA_BINARY_POW = 6,    /* powf(a, b) */
    FCUDA_BINARY_RSUB = 7,   /* b - a */
    FCUDA_BINARY_RDIV = 8,   /* b / a */
    FCUDA_BINARY_RPOW = 9,   /* powf(b, a) */
    FCUDA_BINARY_ATAN2 = 10, /* atan2f(a, b) */
    FCUDA_BINARY_RATAN2 = 11 /* atan2f(b, a) */
};
/* ncnn's BinaryOp operand rule, host only.  Each operand is one image of ncnn rank 1..3 stored as (c, h, w) (rank 2:
 * c = 1; rank 1: c = h = 1).  In this order:
 *   1. equal (c, h, w): the output is that shape;
 *   2. a one-element operand is a scalar: the output is the other operand's shape;
 *   3. a rank-3 blob with a rank-1 operand whose w equals its c broadcasts that operand per channel, as (c, 1, 1): ncnn's
 *      per-channel convention, which wins where numpy alignment would disagree (a rank-1 operand of c values next to a
 *      (c, h, c) blob);
 *   4. otherwise both operands, padded to (c, h, w) with leading 1s, follow numpy's rule on each axis: equal, or 1 on one
 *      side, which broadcasts.
 * The output rank is the larger of the two.  out_shape gets the output (c, h, w); a_aligned and b_aligned get each
 * operand's extent along the output's (c, h, w) axes (the output's extent, or 1 where it broadcasts); the operand's
 * storage read in that shape is unchanged.  -100: a NULL pointer, a rank outside 1..3, a shape entry < 1, or c > 1 with
 * rank < 3, h > 1 with rank 1.  -200: a pair outside the rule. */
int fcuda_binary_op_shape(int a_rank, const int* a_shape, int b_rank, const int* b_shape, int* out_rank, int* out_shape,
                          int* a_aligned, int* b_aligned);
/* out = op(a, b) [then fmaxf(., 0): the Eltwise ReLU, NaN becomes 0] over NCHW fp32 blobs.  a_shape and b_shape are
 * (n, c, h, w); on each of c, h, w the two are equal or one of them is 1, which broadcasts (stride 0) and may be either
 * side; n must be equal.  The output takes the broadcast shape.  With b NULL, b_shape is ignored and every b is
 * b_scalar.  The same-shape ADD is the Eltwise SUM kernel (fcuda_eltwise_add_forward) bit for bit; every other case is
 * one launch of the BinaryOp kernels (profiling kind 6).  output == a is allowed when a broadcasts on no axis, likewise
 * output == b.  Allocates nothing and does not synchronise.
 * -100: NULL output, a or a_shape, b without b_shape, or a size < 1.  -200: op outside 0..11, shapes that do not
 * broadcast, unequal n, an output plane of 2^31 floats or more, or output equal to an operand that broadcasts.  Both are
 * decided before any launch. */
int fcuda_binary_op_forward(float* output, const float* a, const int* a_shape, const float* b, const int* b_shape,
                            float b_scalar, int op, int relu, void* stream);
/* ReluLayer::Forward (src/layers/relu_layer.h:29-41). */
int fcuda_relu_forward(float* output, const float* input, size_t n, void* stream);
/* ncnn's Clip (the reference has no such layer; Caffe's ReLU6 is min 0, max 6): y = min(max(x, min), max) over n
 * floats.  NaN maps to min (ncnn's compare-and-assign passes it through).  -200 for min > max or a NaN bound.  In-place
 * (output == input) is allowed. */
int fcuda_clip_forward(float* output, const float* input, size_t n, float min, float max, void* stream);
/* ncnn's element-wise activation layers (the reference has none; MobileNet-v3, EfficientNet and ESPCN use them), in a
 * numbering of their own: FcudaActivation names the convolution epilogues' activations, which stay 0..2.
 * Definitions, every operation in fp32 and rounded once (IEEE division; no FMA contraction), x the input:
 *   SIGMOID      y = fl(1 / fl(1 + expf(-x)))                      (the statement YOLO's decode uses, bit for bit)
 *   TANH         y = tanhf(x)
 *   SWISH        y = fl(x / fl(1 + expf(-x)))
 *   HARDSIGMOID  y = x < lower ? 0 : x > upper ? 1 : fl(fl(x * alpha) + beta)
 *   HARDSWISH    y = x < lower ? 0 : x > upper ? x : fl(x * fl(fl(x * alpha) + beta))
 * with lower = fl(-beta / alpha) and upper = fl(fl(1 / alpha) + lower), computed once in fp32 on the host as ncnn's
 * load_param does.  ncnn's defaults are alpha 0.2, beta 0.5; PyTorch's hardswish / hardsigmoid are alpha 1/6, beta 0.5,
 * which pnnx writes as 0=1.666667e-01.
 * NaN propagates through every type: both comparisons of the hard types are false for NaN, so it reaches the linear
 * branch.  (Clip differs: fmaxf maps NaN to its min.)  SWISH(-inf) is NaN (-inf / inf), as in ncnn; SWISH(+inf) = +inf.
 * Bounds against the exact value f(x) (float64), from the CUDA C Programming Guide's ulp table (expf and tanhf: 2 ulp;
 * one ulp of v is at most 2^-23 |v|) and 2^-24 relative per rounding:
 *   SIGMOID      |y - f| <= 2^-21 |f| + 2^-126    SWISH  |y - f| <= 2^-21 |f| + 2^-118
 *   TANH         |y - f| <= 2^-22 |f| + 2^-148
 * The relative term is 3 ulp of first order (expf's 2 ulp carried through 1 + e, which does not amplify it, and two
 * roundings), with headroom.  The absolute term covers x below about -87.3, where the true value is subnormal, and below
 * -88.72, where expf(-x) overflows to +inf and SIGMOID / SWISH return +-0 while f is a tiny normal or subnormal
 * (|SWISH| <= 88.8 e^-88.72 < 2^-118 there).  TANH's absolute term is two subnormal spacings.
 * The hard types, against f evaluated in float64 with the same fp32 lower / upper (so the same branch); the 2^-149 terms
 * are the subnormal rounding of products near zero:
 *   HARDSIGMOID  |y - f| <= 2^-23 (|x alpha| + |f|) + 2^-149
 *   HARDSWISH    |y - f| <= 2^-23 (|x| (|x alpha| + |x alpha + beta|) + |f|) + 2^-149 (|x| + 1) */
enum FcudaActivationType {
    FCUDA_ACTIVATION_SIGMOID = 0,
    FCUDA_ACTIVATION_TANH = 1,
    FCUDA_ACTIVATION_SWISH = 2,
    FCUDA_ACTIVATION_HARDSIGMOID = 3,
    FCUDA_ACTIVATION_HARDSWISH = 4,
    FCUDA_ACTIVATION_GELU = 6,
    FCUDA_ACTIVATION_GELU_TANH = 7
};
/* GELU (ncnn's GELU layer; 0=fast_gelu picks the form; Vision Transformers' MLP).  5 stays unassigned and is rejected,
 * so no value that was invalid for the five types above gains a meaning it did not have.
 *   GELU         y = fl(fl(0.5 x) * fl(1 + erff(fl(x * c))))               c = fl(1 / sqrt(2))
 *   GELU_TANH    y = fl(fl(0.5 x) * fl(1 + tanhf(fl(k0 * fl(x + fl(k1 * fl(fl(x * x) * x)))))))
 *                                                                            k0 = fl(sqrt(2 / pi)), k1 = 0.044715f
 * against f = 0.5 x (1 + erf(x / sqrt 2)), resp. 0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3))) in float64 (what
 * torch.nn.GELU computes with approximate 'none' / 'tanh'):
 *   |y - f| <= 2^-21 |x| + 2^-23 |f| + 2^-148        (both forms, finite x)
 * erff and tanhf are 2 ulp (at most 2^-22 for a value of magnitude <= 1); their argument carries <= 7 roundings
 * (k0, k1, c included) of terms of one sign, and the derivative bound |z| (1 - tanh^2 z) <= 0.45 (resp. 1.13 |u|
 * e^-u^2 <= 0.43) keeps the argument's share under 2^-23; 1 + t adds one rounding of <= 2^-23.  Multiplied by 0.5 |x|
 * that is under 2^-21 |x|; the last product adds 2^-24 |f|.  The absolute term covers the loss of 1 + t to cancellation
 * for x far below 0, where f is tiny and y may round to +-0.  NaN propagates. */
/* y = act(x) over n floats, `type` an FcudaActivationType; alpha and beta are read by HARDSIGMOID / HARDSWISH only.  One
 * launch (profiling kind 14).  output == input is allowed.  Allocates nothing and does not synchronise.
 * -100: NULL output or input, or n == 0.  -200: a type that is not an FcudaActivationType, or, for HARDSIGMOID /
 * HARDSWISH, alpha 0 or not finite, or beta not finite.  Both are decided before any launch. */
int fcuda_activation_forward(float* output, const float* input, size_t n, int type, float alpha, float beta,
                             void* stream);
/* ncnn's PReLU (the reference has none): y = x < 0 ? x * slope[c] : x over (batch, channels, plane) with num_slope ==
 * channels slopes, or one slope shared by every channel (num_slope == 1); -200 for any other num_slope.  NaN passes
 * through.  `slope` is a device pointer.  In-place (output == input) is allowed. */
int fcuda_prelu_forward(float* output, const float* input, int channels, size_t plane, const float* slope, int num_slope,
                        int batch, void* stream);
/* ncnn's Normalize (the reference has none; SSD's conv4_3_norm) over (batch, channels, plane).  Per image, the reduction
 * set R is: across_spatial 0 (across_channel must be 1): the `channels` values of one pixel; across_spatial 1,
 * across_channel 1: the whole image; across_spatial 1, across_channel 0: the plane of one channel.  ssum = sum of x^2
 * over R in fp32, and
 *   eps_mode 0 (Caffe / MXNet)  a = 1 / sqrt(ssum + eps)
 *   eps_mode 1 (PyTorch)        a = 1 / max(sqrt(ssum), eps)
 *   eps_mode 2 (TensorFlow)     a = 1 / sqrt(max(ssum, eps))
 * each operation rounded in fp32 (IEEE sqrt and division); then y = fl(fl(x * a) * s_c): the factor first, the scale
 * second, with s_c = scale[0] when num_scale == 1 (shared) or scale[c] when num_scale == channels.  Nothing else is
 * special-cased: an all-zero R gives 0 when eps > 0, and NaN (0 * inf) when eps == 0, in every eps_mode.
 * Summation order (a result depends on its reduction set's values only: the same bits for any batch split, pointer
 * alignment, in or out of place, eager or in a CUDA graph):
 *   per pixel    warp w (0..7) adds the terms of channels w, w + 8, w + 16, ... in increasing order, one fmaf each,
 *                then the eight warp partials are added in warp order;
 *   across_spatial  the set, as one contiguous run of n floats, is cut into chunks of 8192; in a chunk thread t (0..255)
 *                adds the terms of elements t, t + 256, ... in order by fmaf, a 32-lane xor-shuffle tree sums each
 *                warp and the eight warp partials are added in warp order; the chunk sums are added lane-strided (lane
 *                l: chunks l, l + 32, ... in order) and by a 32-lane xor-shuffle tree.
 * The per-pixel mode is one launch that reads the blob once and writes it once (the tile of consecutive pixels stays in
 * shared memory for C <= 1024; past that the write pass re-reads it, from L2) and needs no workspace.  The across_spatial
 * modes take two launches through `workspace`: fcuda_normalize_workspace_size floats, written before they are read.
 * No atomics.  In-place (output == input) is allowed.  Stream-ordered: allocates and synchronises nothing.
 * -100: a NULL pointer (workspace only where its size is not 0), channels, plane or batch < 1.  -200: num_scale other
 * than 1 or channels, eps_mode outside 0..2, across_spatial == across_channel == 0, a negative or NaN eps. */
int fcuda_normalize_workspace_size(int across_spatial, int across_channel, int channels, size_t plane, int batch,
                                   size_t* floats);
int fcuda_normalize_forward(float* output, const float* input, int channels, size_t plane, const float* scale,
                            int num_scale, int across_spatial, int across_channel, float eps, int eps_mode,
                            float* workspace, int batch, void* stream);
/* ncnn's LRN (the reference has none; Caffe's local response normalisation in AlexNet, CaffeNet and GoogLeNet) over
 * (batch, channels, h, w) with dense planes.  r = local_size / 2, sq(v) = fl(v * v), each square rounded on its own.
 *   region_type 0 (ACROSS_CHANNELS)  ss(q, i, j) = sum of sq(x[p][i][j]) for p = max(0, q - r) .. min(C - 1, q + r) in
 *                                    ascending p, one rounded add per term; a = fl(alpha / local_size).
 *   region_type 1 (WITHIN_CHANNEL)   ss(q, i, j) = sum of sq(x[q][i + di][j + dj]) for di = -r .. r (outer) and
 *                                    dj = -r .. r (inner), a term outside the plane being 0; a = fl(alpha / local_size^2).
 * Then s = fl(bias + fl(a * ss)) and y = fl(x * powf(s, -beta)), each operation rounded in fp32 with no contraction and
 * CUDA's full-precision powf.  Nothing is special-cased: s = 0 gives x * inf.  This is the order ncnn's CPU loop adds
 * in, so the only difference from it is powf; a result depends only on the values in its window: the same bits for any
 * batch split, pointer alignment, eager or in a CUDA graph.
 * One launch, no workspace.  ACROSS_CHANNELS reads each input element from HBM once and writes each output once (every
 * thread walks the channels of its pixels through a cp.async ring, 16-byte accesses when h * w % 4 == 0 and both
 * pointers are 16-byte aligned); local_size 1, 3, 5 and 7 are compiled specialisations, larger sizes a generic kernel
 * that reads each window through the cache.  WITHIN_CHANNEL squares a 2D tile and its r-wide halo once in shared memory.
 * Out of place only.  Stream-ordered: allocates and synchronises nothing.
 * -100: a NULL pointer, batch, channels, h or w < 1.  -200: region_type outside 0..1, local_size < 1 or even,
 * output == input. */
int fcuda_lrn_forward(float* output, const float* input, int channels, int h, int w, int region_type, int local_size,
                      float alpha, float beta, float bias, int batch, void* stream);
/* A padding of each (n, c) plane (ncnn's Padding with front = behind = 0; PyTorch's ConstantPad2d, ReplicationPad2d and
 * ReflectionPad2d): top / bottom rows and left / right columns added, all >= 0.  type 0 constant (`value`), 1 replicate
 * (the edge element), 2 reflect (mirrored about the edge, the edge itself excluded: pads < the dimension they pad).
 * Output element (oy, ox) of the (h + top + bottom) x (w + left + right) plane reads input row sy = src(oy, h, top) and
 * column sx = src(ox, w, left), src(o, n, before) = i = o - before when 0 <= i < n, else: constant none (the element
 * is `value`), replicate clamp(i, 0, n - 1), reflect -i when i < 0 and 2 (n - 1) - i when i >= n. */
typedef struct FcudaPad {
    int top, bottom, left, right;
    int type;
    float value;
} FcudaPad;
/* ncnn's InstanceNorm over (batch, channels, h, w) (PyTorch's InstanceNorm2d in eval without running statistics).  Per
 * (n, c) plane of S = h * w floats, in fp32:
 *   mean = sum(x) / S,  var = sum((x - mean)^2) / S  (biased; never E[x^2] - mean^2),
 *   a = gamma[c] / sqrtf(var + eps), or 1 / sqrtf(var + eps) when gamma == beta == NULL (affine 0),
 *   b = fmaf(-mean, a, beta[c]) (beta 0 without affine),
 *   y = fmaf(x, a, b): one fused multiply-add, one rounding; then with `relu` y = fmaxf(y, 0.f) (the ReLU kernel's
 *   expression, so a NaN y gives 0 there too); then, with a non-zero `pad`, the output plane is padded as
 *   fcuda_padding_forward does: border elements are a * x_src + b (with the ReLU) of the element src() maps them to, and
 *   constant borders are `value` with no ReLU.  So IN, then ReLU, then Padding as separate calls give the same bits.
 * IEEE sqrtf and division.  S is converted to float (exact: S <= 2^24).
 * Order (a plane's result depends on its own values only: the same bits for any batch split, pointer offset, in or out
 * of place, eager or in a CUDA graph; the vector width and alignment change loads, never the order):
 *   the plane is cut into chunks of 8192 floats (n_k the size of chunk k, K = ceil(S / 8192) chunks).  In a chunk,
 *   thread t (0..255) adds its elements 4t + 1024j + q (j = 0..7 outer, q = 0..3 inner, those < n_k) in that order
 *   from 0.f, a 32-lane xor-shuffle tree sums each warp and the eight warp partials are added in warp order: sum_k.
 *   m_k = sum_k / n_k, and M2_k = sum of (x - m_k)^2 in the same order, each term one fmaf.  Then lane l (0..31) adds
 *   sum_k for chunks k = l, l + 32, ... in order from 0.f and a 32-lane xor-shuffle tree gives the total: mean = total
 *   / S; lane l adds fmaf(n_k d, d, M2_k) with d = sum_k / n_k - mean over the same chunks, a shuffle tree gives M2 and
 *   var = M2 / S (Chan et al.'s combination).
 * Error bound (first order; float64 quantities of the plane: mean mu, biased variance s2, X = max |x|, A = |a| with
 * the exact mean and variance; U = 2^-24, D = 64 + ceil(K / 32)):
 *   dmu = D U X,  V = (D + 8) U s2 + 4 D U X sqrt(s2) + 6 D^2 U^2 X^2,  rho = V / (s2 + eps) + 6 U,
 *   |y - y64| <= A (rho |x - mu| + (1 + 2 rho) dmu) + U (|beta| + (1 + rho) A (|mu| + dmu) + |y64|)
 * per element before the ReLU and the padding (which change no bound: fmaxf is non-expansive, padding copies).
 * Two launches through `workspace` (fcuda_instance_norm_workspace_size floats: 2 per chunk of every plane, written
 * before they are read), no atomics.  Launch 1 reads each chunk once into registers; launch 2 has one CTA per chunk of
 * the output plane, reads its source elements again and writes them.  Stream-ordered: allocates and synchronises
 * nothing.  In place (output == input) is allowed without a padding.
 * Every launch-2 CTA re-reads its plane's K partials, so a plane costs K * K2 * 8 bytes of workspace reads (K2 the
 * chunks of the output plane); the 2^24-float limits below keep that under 32 MB per plane.
 * -100: a NULL output, input or workspace, exactly one of gamma / beta NULL, channels, h, w or batch < 1.  -200: a
 * negative pad, a type outside 0..2, a reflect pad >= the dimension it pads, a negative or NaN eps, h * w or the padded
 * plane over 2^24 floats, a non-zero pad with output == input.  `pad` NULL or all zero: no padding. */
int fcuda_instance_norm_workspace_size(int channels, size_t plane, int batch, size_t* floats);
int fcuda_instance_norm_forward(float* output, const float* input, int channels, int h, int w, const float* gamma,
                                const float* beta, float eps, int relu, const FcudaPad* pad, float* workspace,
                                int batch, void* stream);
/* ncnn's Padding (front = behind = 0, one pad value) of each (n, c) plane: a pure copy through the index function of
 * FcudaPad, bit-exact; coalesced stores, 16 bytes wide when the padded plane is a multiple of 4 floats and the
 * pointers are 16-byte aligned.  In place (output == input) only with every pad 0.  -100: a NULL pointer (pad
 * included), channels, h, w or batch < 1.  -200: a negative pad, a type outside 0..2, a reflect pad >= the dimension
 * it pads, h * w or the padded plane over 2^31 - 1 floats, a non-zero pad with output == input. */
int fcuda_padding_forward(float* output, const float* input, int channels, int h, int w, const FcudaPad* pad, int batch,
                          void* stream);
/* ncnn's LayerNorm (Vision Transformers): each of `rows` rows of n contiguous floats is normalised over itself,
 *   y = (x - mean) / sqrt(var + eps) * gamma[i] + beta[i]     (i the position in the row; biased variance, eps inside
 * the square root, as torch.nn.LayerNorm).  A rank-2 blob's rows are its h rows (n = w); a rank-3 blob takes n = w
 * (every row of every channel) or n = w * h (every channel plane).  gamma and beta are n floats each, or both NULL.
 * Rounding order (every operation fp32, rounded once; fixed, with no atomics, so the bits do not depend on the batch, the
 * launch geometry or the alignment): one warp per row.  Lane l (0..31) adds x[l + 32 j] for j = 0, 1, ... in order
 * from 0.f; a 32-lane xor-shuffle tree (offsets 16, 8, 4, 2, 1) gives the sum, mean = sum / n.  With d = x - mean,
 * lane l accumulates q = fmaf(d, d, q) over the same elements in the same order and the same tree gives Q; var = Q / n,
 * r = __frsqrt_rn(var + eps), y = fmaf(d * r, gamma, beta) (y = d * r without gamma / beta).  Rows of at most 1024
 * floats are read once into registers; longer rows are read again for each pass.
 * Error bound (first order; float64 quantities of the row: mean mu, biased variance s2, sigma = sqrt(s2 + eps),
 * M = mean |x|, U = 2^-24, L = ceil(n / 32) + 5 the length of the longest addition chain):
 *   e = (L + 1) U M,   rho = (L + 6) U + (e / sigma)^2,
 *   |y - y64| <= |gamma| (rho |x - mu| + (1 + rho) e) / sigma + 2^-23 (|y64| + |gamma| |x - mu| / sigma) + 2^-149
 * (gamma = 1, beta = 0 without the affine).  One launch (profiling kind 16).  output == input is allowed.  Allocates
 * nothing and does not synchronise.  -100: a NULL output or input, n or rows < 1.  -200: exactly one of gamma / beta
 * NULL, eps negative or not finite.  Both are decided before any launch. */
int fcuda_layer_norm_forward(float* output, const float* input, int n, long long rows, const float* gamma,
                             const float* beta, float eps, void* stream);
/* Scaled dot-product attention of ncnn's MultiHeadAttention (torch.nn.MultiheadAttention without a mask or dropout),
 * after the input projections and before the output projection.  Q, K and V are row-major fp32 buffers
 * [batch][Lq or Lk][ld]; head h of image b reads columns h * d .. h * d + d - 1 of its rows (ldq / ldk / ldv in floats,
 * so one [N L][3E] buffer of a fused QKV projection is read in place with ld = 3E).  O is [batch][Lq][heads * d]:
 *   O[b][i][h d + c] = sum_j softmax_j(scale * Q_i . K_j) V[j][c]   over the keys j < Lk of image b, head h.
 * One CTA (128 threads) per (image, head, 64-query tile); it walks the key tiles of 64 in order.  S = Q K^T and O = P V
 * run on wgmma in BF16x3 (each operand x = p1 + p2 + r, |r| <= 2^-16 |x|, three bf16 products p2 q1 + p1 q2 + p1 q1 into
 * fp32): Q and P are split in registers, K and V as they are staged into shared memory.  The softmax is online in fp32:
 * s = fl(S scale), running max m, p = expf(s - m), the running sum l and O rescaled by expf(m_old - m_new) per tile,
 * O / l once at the end.  Key tails are masked to -inf (their K and V staged as 0); query tails are not stored.  The
 * bits do not depend on how the batch is split across calls.
 * Error bound against float64 attention of the same fp32 Q, K, V (per element; U = 2^-24, T = ceil(Lk / 64) key tiles,
 * s*_ij = scale Q_i . K_j and m*_i = max_j s*_ij in float64, p*_ij = exp(s*_ij - m*_i), a_ij = sum_c |Q_ic| |K_jc|,
 * W_ic = sum_j p*_ij |V_jc| / sum_j p*_ij):
 *   D_i   = max_j ( |scale| a_ij (2^-14 + (d + 1) 2^-21) + (T + 1) U |s*_ij - m*_i| )
 *   eta_i = 2.01 ( D_i + (T + 1) 2^-22 + (2 T + 18) U )
 *   |O_ic - O*_ic| <= ( 2.01 eta_i + 2^-14 + (3 Lk + 3 T + 1) 2^-23 ) W_ic + 2^-126
 * D_i bounds the error of each exponent's argument: the BF16x3 product drops p2 q2 and the residuals (<= 3 2^-16 +
 * O(2^-24) of a_ij), the tensor core accumulates 3 d products in fp32 (<= 2^-23 each, counted as d 2^-21 with
 * headroom), s and s - m round once each, and the running maxima differ by at most max |s - m| per rescale.  eta_i
 * bounds the relative error of each weight p: exp of the argument error, expf's 2 ulp per p and per rescale, and the
 * fp32 row sum l (a chain of at most 2 T + 18 additions).  A softmax of weights with relative errors <= eta moves the
 * convex combination by at most 2 eta / (1 - eta) W.  The P V product adds the BF16x3 terms of P and V (2^-14) and the
 * fp32 accumulation of 3 Lk products, T rescales and the final division.  expf's 2 ulp is the CUDA C Programming
 * Guide's bound.  This bound is derived, not measured.
 * Allocates nothing and does not synchronise, so it can be captured in a CUDA graph.  One launch (profiling kind 15);
 * images go on grid x (no 65535 cap), heads and query tiles on y.
 * -100: a NULL pointer, batch, heads, Lq or Lk < 1.  -200: d not a multiple of 16 in 16..128, an ld below heads * d, o
 * overlapping q, k or v, heads * ceil(Lq / 64) over 65535, or a scale that is 0 or not finite.  Both are decided before
 * any launch. */
int fcuda_attention_forward(float* o, const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                            int batch, int heads, int d, int lq, int lk, float scale, void* stream);
/* SoftmaxLayer::Forward (src/layers/softmax_layer.h:32-55): over each image's whole blob. */
int fcuda_softmax_forward(float* output, const float* input, size_t n_per_image, int batch, void* stream);
/* DropoutLayer::Forward (src/layers/dropout_layer.h:36-57): y = x*scale (copy when scale == 1). */
int fcuda_dropout_forward(float* output, const float* input, size_t n, float scale, void* stream);
/* ConcatLayer / SplitLayer copies (src/layers/concat_layer.h:37-47, split_layer.h:43-53): copies `channels`
 * channels of every image into dst at channel offset `dst_channel_offset` of a dst with `dst_channels`. */
int fcuda_copy_channels(float* dst, int dst_channels, int dst_channel_offset, const float* src, int channels,
                        size_t stride, int batch, void* stream);

/* fcuda_conv_forward_opts with only residual / relu_after_add set; -100 for a NULL residual. */
int fcuda_conv_forward_residual(const FcudaConvParam* param, int algo, float* output, const float* input,
                                const float* packed_kernel, float* scratch, const float* bias, const float* residual,
                                int relu_after_add, int batch, void* stream);

/* Whether the algorithm can apply FcudaConvOptions::pool in its epilogue (Winograd F(6,3)/F(2,3): the output tile is pooled
 * in registers; FCUDA_SGECONV: 3x3 / stride-1 layers with IC % 32 == 0, pooled by two shuffles per value). */
int fcuda_conv_can_pool(const FcudaConvParam* param, int algo);

/* FCUDA_SGECONV in the current arithmetic mode: 1 when the layer (output_h / output_w assigned) runs on the halo kernel
 * (switch igemm_halo below: stride 1, no dilation, more than one tap, input_channels / group % 32 == 0, input_w % 4 == 0,
 * 16-byte aligned input), with geom[0..3] = output patch rows, patch columns, shared-memory box rows, box columns;
 * 0 when it keeps the gathering kernel.  The switch itself is not consulted. */
int fcuda_igemm_halo_tile(const FcudaConvParam* param, int* geom);
/* The same for the pre-split halo kernel (switch igemm_presplit below; fp32split mode only): 1 when the layer runs on it,
 * with geom[0..3] = tile rows, tile columns (rows * columns = 128), fp32 box rows, box columns; 0 otherwise.  The switch
 * itself is not consulted. */
int fcuda_igemm_presplit_tile(const FcudaConvParam* param, int* geom);
/* The same for the wide pre-split kernel (switch igemm_wide below), which takes a layer of the pre-split kernel whose N
 * tile is 64 or 128 output channels, with at least 5 taps, where its tile pads no more pixels than the pre-split patch:
 * 1 with geom[0..3] = tile rows (28), tile columns (16 for a 64-channel N tile, 8 for 128), fp32 box rows, box columns;
 * 0 otherwise.  The switches themselves are not consulted. */
int fcuda_igemm_wide_tile(const FcudaConvParam* param, int* geom);
/* FCUDA_SGECONV in the current arithmetic mode: 1 when the layer (output_h / output_w assigned) with `options` (NULL = the
 * all-zero struct) runs on the persistent stem kernel (switch igemm_stem below: fp32split mode, input_channels / group
 * % 32 != 0, kernel_h * kernel_w * input_channels / group <= 256, output_channels / group <= 128, no residual, pooling or
 * dilation); 0 when it keeps the gathering kernel.  The switch itself is not consulted. */
int fcuda_igemm_stem_supported(const FcudaConvParam* param, const FcudaConvOptions* options);
/* fcuda_conv_forward_opts with only pool set. */
int fcuda_conv_forward_pool(const FcudaConvParam* param, int algo, float* output, const float* input,
                            const float* packed_kernel, float* scratch, const float* bias, int batch, void* stream);

/* Input staging on the GPU, the step before the hot path (SURVEY.md §8f rank 3).  One fused pass over a batch of u8 images:
 * ncnn::Mat::from_pixels / from_pixels_resize (src/ncnn/mat.h:149-152; mat_pixel.cpp:1329-1410; the 11-bit fixed-point
 * bilinear of mat_pixel_resize.cpp:26-278, bit-exact) and Mat::substract_mean_normalize (mat.h:159-160, mat.cpp:30-107).
 *   type       ncnn pixel type, mat.h:126-146: PIXEL_RGB 1, BGR 2, GRAY 4, RGBA 8, conversions = from | (to << 16)
 *   pixels     DEVICE pointer, `batch` interleaved u8 images of w*h*src_channels bytes each
 *   target_*   output size (<= 0: keep w / h; equal to w / h: no resize, like mat_pixel.cpp:1371)
 *   mean/norm  HOST arrays of out_channels floats or NULL (mean only: x - mean; norm only: x * norm; both: x*norm - mean*norm)
 *   output     (batch, out_channels, target_h, target_w) fp32, dense planes
 * Returns -200 for a type from_pixels does not know (it returns an empty Mat). */
int fcuda_pixel_channels(int type, int* src_channels, int* out_channels);
int fcuda_from_pixels(float* output, const unsigned char* pixels, int type, int w, int h, int target_w, int target_h,
                      const float* mean_vals, const float* norm_vals, int batch, void* stream);

/* fcuda_conv_forward_opts with only residual / relu_after_add (`residual` may be NULL) and the dilations set; -100 for a
 * dilation < 1.
 * Groups (the reference rejects partial groups, avx/booster.cpp:304-308): with FCUDA_SGECONV and param->group > 1, through
 * every entry point, input_channels and output_channels are the TOTAL channel counts, the raw kernel is
 * (OC, IC/group, KH, KW) and group g maps input channels [g*IC/G, (g+1)*IC/G) to output channels [g*OC/G, (g+1)*OC/G). */
int fcuda_conv_forward_ext(const FcudaConvParam* param, int algo, float* output, const float* input,
                           const float* packed_kernel, float* scratch, const float* bias, const float* residual,
                           int relu_after_add, int dilation_h, int dilation_w, int batch, void* stream);

/* ncnn's Deconvolution / DeconvolutionDepthWise (transposed convolution; the reference has no such layer).  Weights are
 * (OC, IC/group, KH, KW) as ncnn stores them (group-major, not flipped); channel counts are TOTAL counts.  With
 *   Hf = (H-1)*stride_h + dilation_h*(KH-1) + 1 + output_pad_bottom     (Wf likewise with output_pad_right)
 *   full[n][oc][Y][X] = bias[oc] + sum of x[n][ic][i][j] * w[oc][ic - g0][ky][kx] over ic in oc's group and
 *                       i*stride_h + ky*dilation_h = Y, j*stride_w + kx*dilation_w = X
 * the output is act(full) cropped by the four pads: output_h = Hf - pad_top - pad_bottom (output_w likewise).
 * Rejected with -200: a negative pad or output pad, activation other than none / ReLU, stride > 1 together with
 * dilation > 1 in one direction, OC or IC not divisible by group.  -100 for empty sizes or an empty output.
 * How it runs (fcuda_deconv_plan):
 *   group == IC == OC > 1  a CUDA-core gather kernel, one output per thread, taps in ascending (ky, kx) order;
 *   stride 1               the flipped filter as a stride-1 convolution (dilation kept) that writes the output directly
 *                          with bias and ReLU, when every pad is <= dilation*(K-1) and output_pad <= the pad on its side;
 *   otherwise              one stride-1 convolution with OC' = stride_h*stride_w*OC channels ordered
 *                          (group, Y % stride_h, X % stride_w, oc in group) and kernel ceil(K/stride) (the sub-pixel
 *                          phases of the filter), pads (kernel-1)*dilation, into scratch; then a scatter kernel adds the
 *                          bias once, applies the ReLU and writes the cropped output. */
typedef struct FcudaDeconvParam {
    int output_channels, input_channels, input_h, input_w, kernel_h, kernel_w, stride_h, stride_w, dilation_h, dilation_w,
        pad_left, pad_right, pad_top, pad_bottom, output_pad_right, output_pad_bottom, group, bias_term, activation,
        output_h, output_w;
} FcudaDeconvParam;
/* Validates the parameters and fills output_h / output_w. */
int fcuda_deconv_output_dim(FcudaDeconvParam* param);
/* The equivalent convolution (output_h / output_w assigned) and the algorithm it runs with: fcuda_conv_select_algo_tuned,
 * except FCUDA_SGECONV with dilation or with group > 1.  FCUDA_DEPTHWISE means the gather kernel; `equivalent` is then
 * zeroed.  Either output pointer may be NULL. */
int fcuda_deconv_plan(const FcudaDeconvParam* param, FcudaConvParam* equivalent, int* conv_algo);
/* Scratch for `batch` images: the equivalent convolution's scratch (rounded up to 64 floats) plus
 * batch * OC' * Hc * Wc floats for its output on the sub-pixel path; packed = the equivalent convolution's packed filter
 * (IC*KH*KW floats for the gather kernel). */
int fcuda_deconv_get_buffer_size(const FcudaDeconvParam* param, int batch, size_t* scratch_floats, size_t* packed_floats);
/* Builds the equivalent filter from the raw weights (host or device pointer) and packs it like fcuda_conv_init.  Synchronous. */
int fcuda_deconv_init(const FcudaDeconvParam* param, float* packed, const float* raw, void* stream);
/* output (batch, OC, output_h, output_w) <- input (batch, IC, H, W).  `bias` is OC floats, or NULL when !bias_term.
 * Allocates nothing and does not synchronise. */
int fcuda_deconv_forward(const FcudaDeconvParam* param, float* output, const float* input, const float* packed,
                         float* scratch, const float* bias, int batch, void* stream);

/* ncnn's Interp (the reference has no such layer; its unused caffe_cpu_interp2 maps src = dst * in / out, which is neither
 * ncnn mode): input (batch, C, input_h, input_w) -> output (batch, C, output_h, output_w).
 *   resize_type 1 nearest:  hs = output_height ? input_h / (float)output_h : 1.f / height_scale (fp32, ws likewise),
 *                           source row min((int)(y * hs), input_h - 1); a pure gather, bit-exact.
 *   resize_type 2 bilinear: scales from the sizes.  align_corner 0 (half pixel): fy = (y + 0.5) * input_h / output_h - 0.5,
 *                           negative fy clamped to 0; align_corner 1: fy = y * (input_h - 1) / (output_h - 1), 0 when
 *                           output_h == 1.  Neighbours y0 = (int)fy, y1 = min(y0 + 1, input_h - 1), weight fy - y0; x
 *                           likewise; interpolated horizontally on both rows, then vertically (PyTorch's
 *                           F.interpolate(mode="bilinear", align_corners=...) definition).
 * Equal input and output sizes (and, for nearest, hs == ws == 1) are a straight copy.
 * Rejected with -200: resize_type other than 1 / 2 (bicubic is not built).  -100: empty input or output, or a
 * non-positive scale where a scale is used. */
typedef struct FcudaInterpParam {
    int resize_type, align_corner;
    float height_scale, width_scale;
    int output_height, output_width; /* explicit size; when either is 0 both come from the scales */
    int input_h, input_w;
    int output_h, output_w;          /* filled by fcuda_interp_output_dim */
} FcudaInterpParam;
/* Validates the parameters and fills output_h / output_w: output_height / output_width when both are set, otherwise
 * (int)(input_h * height_scale) and (int)(input_w * width_scale) with fp32 products, as ncnn computes them. */
int fcuda_interp_output_dim(FcudaInterpParam* param);
/* output <- input for `channels` planes of each of `batch` images.  Allocates nothing and does not synchronise. */
int fcuda_interp_forward(const FcudaInterpParam* param, float* output, const float* input, int channels, int batch,
                         void* stream);
/* ncnn's PixelShuffle (sub-pixel convolution upsampling; the reference has no such layer): input (batch, C, h, w) ->
 * output (batch, C / r^2, h * r, w * r), with OC = C / r^2 and output element (p, y, x), y = h' * r + i, x = w' * r + j
 * (0 <= i, j < r), read from input channel
 *   mode 0:  q = p * r^2 + i * r + j      (PyTorch's nn.PixelShuffle, ONNX DepthToSpace CRD)
 *   mode 1:  q = (i * r + j) * OC + p     (ONNX DepthToSpace DCR, TensorFlow's depth_to_space)
 * at (h', w').  Without an addend this is a pure copy, bit-exact, NaN payloads included.
 * With `addend` (batch, OC, addend_map->input_h, addend_map->input_w), each output element becomes
 *   out = shuffled + addend[n][p][min((int)(y * hs), input_h - 1)][min((int)(x * ws), input_w - 1)],
 * one fp32 add (round to nearest), hs / ws the fp32 scales fcuda_interp_forward derives from `addend_map`: the bits of
 * PixelShuffle, then a nearest Interp of the addend, then an Eltwise SUM of the two (fp32 addition commutes, so either
 * bottom order), as three calls.  A NaN sum is the canonical NaN, as the Eltwise kernel writes it.
 * One launch through the deconvolution's sub-pixel scatter kernel (profiling kind 13); it reads the input and the
 * addend once and writes the output once.  Allocates nothing and does not synchronise.
 * -100: a NULL output or input, an addend without addend_map, C, h, w or batch < 1, or an addend_map that
 * fcuda_interp_output_dim rejects with -100.  -200: r < 1, mode other than 0 or 1, C % r^2 != 0, an output plane over
 * 2^31 - 1 floats, output == input or output == addend, an addend_map that is not nearest (resize_type 1) or whose
 * output size is not (h * r, w * r). */
int fcuda_pixel_shuffle_forward(float* output, const float* input, int channels, int h, int w, int r, int mode,
                                const float* addend, const FcudaInterpParam* addend_map, int batch, void* stream);
/* ncnn / Caffe Crop: output (batch, out_c, out_h, out_w)[n][c][y][x] = input (batch, channels, in_h, in_w)
 * [n][c + coff][y + hoff][x + woff].  -100 for empty sizes, a negative offset or a window outside the input.  Allocates
 * nothing and does not synchronise. */
int fcuda_crop_forward(float* output, const float* input, int channels, int in_h, int in_w, int coff, int hoff, int woff,
                       int out_c, int out_h, int out_w, int batch, void* stream);

/* ---- SSD detection head (the reference has none of these layers) ---------------------------------------------------
 * Every call below is stream-ordered: none allocates, synchronises or copies to the host, so all may be captured in a
 * CUDA graph.  -100: a NULL pointer or an empty size; -200: a parameter outside the documented limits. */

/* ncnn's Permute of `batch` (c, h, w) images.  Output (c', h', w') by order_type: 0 (c,h,w), 1 (c,w,h), 2 (h,c,w),
 * 3 (h,w,c), 4 (w,c,h), 5 (w,h,c); -200 for any other order.  A pure gather, bit-exact.  Order 3 (NCHW -> NHWC, SSD's
 * head layout) is a shared-memory tiled transpose with coalesced reads and writes. */
int fcuda_permute_forward(float* output, const float* input, int c, int h, int w, int order_type, int batch, void* stream);

/* Max-subtracted softmax over the middle axis of each of `batch` (outer, len, inner) views:
 * y = expf(x - max) / sum(expf(x - max)).  inner == 1 (SSD's class axis) takes one warp per row of len values.
 * fcuda_softmax_forward (the whole-blob softmax) is a separate kernel. */
int fcuda_softmax_axis_forward(float* output, const float* input, int outer, int len, int inner, int batch, void* stream);

/* Caffe / ncnn PriorBox.  Per location (x, y) of a feat_w x feat_h map, centre ((x + offset) * step_w,
 * (y + offset) * step_h), a step <= 0 meaning img / feat; for each min size in order: the min x min box, then the
 * sqrt(min * max) square if max sizes are given (one per min size), then for each aspect ratio ar (an ar within 1e-6 of 1
 * is skipped) the (min * sqrt(ar), min / sqrt(ar)) box followed by its flip (min / sqrt(ar), min * sqrt(ar)) when `flip`.
 * A box of width bw, height bh is ((cx - bw/2) / img_w, (cy - bh/2) / img_h, (cx + bw/2) / img_w, (cy + bh/2) / img_h),
 * each operation rounded in fp32, clamped to [0, 1] when `clip`.
 * Output: 2 rows of 4 * P floats (P = feat_w * feat_h * per-location count): row 0 the boxes, row 1 the variances.
 * Limits (else -200): 1..16 min sizes, 0 or as many max sizes each > its min size, 0..16 aspect ratios > 0, min sizes > 0,
 * P < 2^24. */
#define FCUDA_PRIORBOX_MAX 16
typedef struct FcudaPriorBoxParam {
    int num_min_sizes, num_max_sizes, num_aspect_ratios;
    float min_sizes[FCUDA_PRIORBOX_MAX], max_sizes[FCUDA_PRIORBOX_MAX], aspect_ratios[FCUDA_PRIORBOX_MAX];
    float variances[4];
    int flip, clip;
    float step_w, step_h; /* <= 0: img / feat */
    float offset;
} FcudaPriorBoxParam;
/* Validates the parameters and gives the number of priors per location. */
int fcuda_priorbox_per_location(const FcudaPriorBoxParam* param, int* per_location);
int fcuda_priorbox_forward(float* output, const FcudaPriorBoxParam* param, int feat_w, int feat_h, int img_w, int img_h,
                           void* stream);

/* SSD centre-size decode (ncnn / Caffe, no clipping) of `batch` images.  loc: (batch, num_priors * 4); priors: the
 * PriorBox output (2, num_priors * 4), shared by every image; boxes: (batch, num_priors * 4) as (xmin, ymin, xmax, ymax).
 *   pw = p2 - p0, ph = p3 - p1, pcx = (p0 + p2) * 0.5, pcy = (p1 + p3) * 0.5
 *   cx = var0 * l0 * pw + pcx, cy = var1 * l1 * ph + pcy, w = expf(var2 * l2) * pw, h = expf(var3 * l3) * ph
 *   box = (cx - w * 0.5, cy - h * 0.5, cx + w * 0.5, cy + h * 0.5)
 * every operation rounded in fp32 left to right (no FMA).  The boxes DetectionOutput uses are these bits. */
int fcuda_ssd_decode(float* boxes, const float* loc, const float* priors, int num_priors, int batch, void* stream);

/* ncnn's DetectionOutput with a fixed-shape output.  conf: (batch, P * C), class fastest; class 0 is background.
 * For each image and class c >= 1: the candidates are the priors with score > conf_threshold, ordered by (score
 * descending, prior ascending), the first nms_top_k kept; then greedy NMS over them in that order: a candidate is kept
 * iff no earlier kept box has IoU > nms_threshold, where for boxes a (the kept one) and b, in fp32, each operation rounded:
 *   area   = (x1 - x0) * (y1 - y0)
 *   iw     = min(a.x1, b.x1) - max(a.x0, b.x0), then 0 if negative     (ih likewise with y)
 *   inter  = iw * ih
 *   union  = (area_b + area_a) - inter
 *   IoU    = inter / union                       a NaN IoU (0 / 0 of two empty boxes) suppresses nothing.
 * The kept boxes of all classes are merged, ordered by (score descending, class ascending, prior ascending), and the first
 * keep_top_k written.  Scores compare as floats: -0 and +0 are equal (ordered by class, then prior), and the row carries
 * the score's own bits.  output: (batch, keep_top_k, 6) rows [label, score, xmin, ymin, xmax, ymax] with the boxes of
 * fcuda_ssd_decode; rows past an image's count are [-1, 0, 0, 0, 0, 0].
 * Limits (else -200): 1 <= nms_top_k <= 1024, 1 <= keep_top_k <= 1024, 1 <= C <= 1024, 1 <= P < 2^24, batch <= 65535,
 * nms_threshold not NaN.  `workspace` holds fcuda_detection_output_workspace_size floats, 8-byte aligned (else -100). */
int fcuda_detection_output_workspace_size(int num_priors, int num_classes, int nms_top_k, int batch, size_t* floats);
int fcuda_detection_output_forward(float* output, const float* loc, const float* conf, const float* priors, int num_priors,
                                   int num_classes, float conf_threshold, float nms_threshold, int nms_top_k, int keep_top_k,
                                   float* workspace, int batch, void* stream);

/* ---- YOLO detection head (the reference has none of these layers) --------------------------------------------------
 * ncnn's YoloDetectionOutput (YOLOv2, version 2) and Yolov3DetectionOutput (version 3), with a fixed-shape output.
 * Stream-ordered like the SSD calls above: nothing allocates, synchronises or copies to the host.
 *
 * Inputs: one (batch, num_box * (5 + C), h, w) blob per scale b (exactly one for version 2), in mask-group order; for box
 * pp the channels pp * (5 + C) + {0: x, 1: y, 2: w, 3: h, 4: objectness, 5..: class logits}.  A slot is one (scale, box,
 * row, column) in that order (ncnn's gather order); slots = sum over scales of num_box * h * w.
 *
 * Decode of the cell (i, j) of box pp on scale b, in fp32, every operation rounded on its own (no FMA), s(t) =
 * 1 / (1 + expf(-t)):
 *   cx = (j + s(x)) / w, cy = (i + s(y)) / h, bw = expf(tw) * bias_w / norm_w, bh = expf(th) * bias_h / norm_h,
 *   box = (cx - bw * 0.5, cy - bh * 0.5, cx + bw * 0.5, cy + bh * 0.5)
 *   version 3: k = mask[b * num_box + pp], bias = (biases[2k], biases[2k + 1]) in input pixels, norm_w =
 *     (int)(anchors_scale[b] * w) (fp32 product, truncated), norm_h likewise.  class = the argmax of the raw logits
 *     (strict >, from -FLT_MAX, so the first maximum wins; all -inf / NaN logits give class 0 with -FLT_MAX), and
 *       confidence = 1 / (1 + expf(-obj) * (1 + expf(-logit_max)))
 *     which is ncnn's expression as written.  ncnn's comment calls it s(obj) * s(logit_max), but the parentheses make it
 *     a different function; it is kept because thresholds shipped with ncnn models were tuned against it.
 *   version 2: bias = (biases[2pp], biases[2pp + 1]) in grid cells, norm_w = w, norm_h = h.  p = the max-subtracted
 *     softmax of the C logits, p_k = expf(l_k - max) / sum (sum in class order), computed without writing the input
 *     (ncnn's layer overwrites its bottom); class = the argmax of p (strict >, from 0), confidence = s(obj) * p_class.
 * A slot is a candidate iff confidence >= confidence_threshold (>=, where SSD's DetectionOutput takes >).
 *
 * Selection, NMS and output: the candidates of each image are ordered by (confidence descending, slot ascending) and the
 * first nms_top_k kept; then one greedy class-agnostic NMS over them in that order: a candidate is kept iff no earlier kept
 * box has IoU > nms_threshold, the IoU being DetectionOutput's above (areas from the corners; a NaN IoU suppresses
 * nothing).  output: (batch, keep_top_k, 6), rows [class + 1, confidence, xmin, ymin, xmax, ymax] in kept order (the + 1
 * is ncnn's prepended background label), then [-1, 0, 0, 0, 0, 0].  ncnn's output has one row per kept box and no cap, so
 * with nms_top_k = keep_top_k = 1024 the rows equal ncnn's whenever at most 1024 slots pass the threshold; past that
 * the lowest-ranked candidates are dropped before NMS, and past keep_top_k kept boxes the rest are dropped.
 *
 * Limits (else -200): version 2 or 3; 1 <= num_class <= 1024; 1 <= num_box <= 16; 1..4 scales (1 for version 2);
 * num_biases <= 128, and >= 2 * num_box for version 2; version 3: every mask index k in 0 <= k < num_biases / 2, and
 * on every scale anchors_scale > 0 with anchors_scale * (the longer grid side) < 2^31 in fp32; slots < 2^24;
 * 1 <= nms_top_k, keep_top_k <= 1024; batch <= 65535; nms_threshold not NaN.  -100: a NULL pointer, batch < 1, a grid
 * side < 1, or a workspace that is not 16-byte aligned (fcuda_yolo_detection_forward). */
#define FCUDA_YOLO_MAX_SCALES 4
#define FCUDA_YOLO_MAX_BOXES 16
#define FCUDA_YOLO_MAX_BIASES 128
typedef struct FcudaYoloParam {
    int version;                                           /* 2: YoloDetectionOutput, 3: Yolov3DetectionOutput */
    int num_class, num_box, num_scales;
    float confidence_threshold, nms_threshold;
    int nms_top_k, keep_top_k;
    int num_biases;                                        /* floats in biases */
    float biases[FCUDA_YOLO_MAX_BIASES];
    int mask[FCUDA_YOLO_MAX_SCALES * FCUDA_YOLO_MAX_BOXES]; /* version 3: num_box per scale */
    float anchors_scale[FCUDA_YOLO_MAX_SCALES];            /* version 3 */
    int grid_h[FCUDA_YOLO_MAX_SCALES], grid_w[FCUDA_YOLO_MAX_SCALES];
} FcudaYoloParam;
/* Decode alone: for every slot of every image, scores (batch, slots) the confidence, classes (batch, slots) the class
 * (without the + 1) and boxes (batch, slots, 4), whether or not the slot is a candidate.  The boxes and confidences
 * fcuda_yolo_detection_forward uses are these bits.  inputs: num_scales device pointers. */
int fcuda_yolo_decode(float* scores, int* classes, float* boxes, const float* const* inputs, const FcudaYoloParam* param,
                      int batch, void* stream);
/* Workspace in floats: batch * (6 * slots + 39937). */
int fcuda_yolo_detection_workspace_size(const FcudaYoloParam* param, int batch, size_t* floats);
int fcuda_yolo_detection_forward(float* output, const float* const* inputs, const FcudaYoloParam* param, float* workspace,
                                 int batch, void* stream);

/* ---- Faster R-CNN and R-FCN: Proposal, ROIPooling and PSROIPooling (the reference has none of them) ----------------
 * Stream-ordered like the detection calls above: nothing allocates, synchronises or copies to the host.
 *
 * Proposal (ncnn's layer, py-faster-rcnn's proposal_layer.py arithmetic) in fp32, every operation rounded on its own (no
 * FMA).  A = 9 anchors, q = ratio * 3 + scale over ratios {0.5, 1, 2} and scales {8, 16, 32}:
 *   rw = roundf(base_size / sqrtf(ratio)), rh = roundf(rw * ratio)       (half away from zero)
 *   aw = rw * scale, ah = rh * scale, ax1 = base_size * 0.5 - aw * 0.5, ay1 = base_size * 0.5 - ah * 0.5
 * With the defaults (ax1, ay1, ax1 + aw - 1, ay1 + ah - 1) is py-faster-rcnn's anchor table.
 * Inputs, per image of `batch`: score (2A, H, W), the foreground score of anchor q at channel A + q; bbox (4A, H, W),
 * channels 4q + {0: dx, 1: dy, 2: dw, 3: dh}; im_info 3 floats (height, width, scale).  Decode of anchor q at cell (y, x):
 *   ax = ax1 + x * feat_stride, ay = ay1 + y * feat_stride
 *   pcx = (ax + aw * 0.5) + aw * dx, pcy likewise, pw = aw * expf(dw), ph = ah * expf(dh)
 *   box = (pcx - pw * 0.5, pcy - ph * 0.5, pcx + pw * 0.5, pcy + ph * 0.5), each x clipped as fmaxf(fminf(x, width - 1), 0)
 *   and each y with height - 1.
 * A box is a candidate iff x2 - x1 + 1 >= min_size * scale, y2 - y1 + 1 >= min_size * scale and its score is not NaN.
 * The candidates are ordered by (score descending, index ascending), index = q * H * W + y * W + x (-0 and +0 are equal
 * scores), and the first pre_nms_topN kept; then greedy NMS in that order: a candidate is kept iff no earlier kept box has
 * IoU > nms_thresh, with the + 1 pixel convention:
 *   iw = fmaxf((min(x2) - max(x1)) + 1, 0), ih likewise, inter = iw * ih, area = (x2 - x1 + 1) * (y2 - y1 + 1)
 *   IoU = inter / ((area_a + area_b) - inter)                a NaN IoU suppresses nothing
 * and it stops at after_nms_topN kept boxes.  rois: (batch, after_nms_topN, 4) rows [x1, y1, x2, y2] in kept order, then
 * [0, 0, 0, 0]; scores (may be NULL): (batch, after_nms_topN), the kept boxes' score bits, then -1.
 * Limits (else -200): feat_stride, base_size >= 1; 1 <= pre_nms_topN, after_nms_topN <= 8192; nms_thresh not NaN;
 * A * H * W < 2^24; batch <= 65535.  -100: a NULL pointer, batch < 1, H or W < 1, or a workspace that is not 16-byte
 * aligned (fcuda_proposal_forward). */
#define FCUDA_PROPOSAL_ANCHORS 9
typedef struct FcudaProposalParam {
    int feat_stride, base_size;      /* ncnn 0= (16), 1= (16) */
    int pre_nms_topN, after_nms_topN; /* 2= (6000), 3= (300) */
    float nms_thresh;                 /* 4= (0.7) */
    int min_size;                     /* 5= (16) */
} FcudaProposalParam;
/* The 9 anchors as (ax1, ay1, aw, ah) rows, anchor q at table[4q..4q+3]; host only, after the limits above. */
int fcuda_proposal_anchors(const FcudaProposalParam* param, float* table);
/* Decode alone: boxes (batch, A * H * W, 4), clipped, for every anchor and cell whether or not it is a candidate.  The
 * boxes fcuda_proposal_forward uses are these bits. */
int fcuda_proposal_decode(float* boxes, const float* score, const float* bbox, const float* im_info,
                          const FcudaProposalParam* param, int feat_h, int feat_w, int batch, void* stream);
/* Workspace in floats: with P = 9 * H * W, K = pre_nms_topN and r4(v) = v rounded up to a multiple of 4,
 * batch * (4 P + r4(P) + 4 K + 2 r4(K) + K * ceil(K / 32)) + r4(batch). */
int fcuda_proposal_workspace_size(const FcudaProposalParam* param, int feat_h, int feat_w, int batch, size_t* floats);
int fcuda_proposal_forward(float* rois, float* scores, const float* score, const float* bbox, const float* im_info,
                           const FcudaProposalParam* param, int feat_h, int feat_w, float* workspace, int batch,
                           void* stream);

/* ROIPooling (Caffe's and ncnn's arithmetic): input (batch, C, H, W), rois (batch, num_rois, 4) [x1, y1, x2, y2] in input
 * pixels; output (batch * num_rois, C, pooled_h, pooled_w), RoI r of image n at item n * num_rois + r pooling image n.
 *   x1 = (int)roundf(roi[0] * spatial_scale), likewise y1, x2, y2 (half away from zero, converted saturating)
 *   roi_w = max(x2 - x1 + 1, 1), bin_w = (float)roi_w / pooled_w      (roi_h, bin_h likewise)
 *   wstart = floorf(pw * bin_w) + x1, wend = ceilf((pw + 1) * bin_w) + x1, both clamped to [0, W]   (h likewise)
 *   value = 0 for an empty bin, else the fmaxf over the bin from -FLT_MAX: bit-exact.
 * Limits: -200 for pooled_w or pooled_h < 1 or spatial_scale not finite and > 0; -100 for a NULL pointer or a size < 1.
 * Every RoI row is pooled, the [0, 0, 0, 0] padding of fcuda_proposal_forward included. */
int fcuda_roi_pooling_forward(float* output, const float* input, const float* rois, int channels, int height, int width,
                              int num_rois, int pooled_h, int pooled_w, float spatial_scale, int batch, void* stream);

/* PSROIPooling (R-FCN's position-sensitive RoI average pooling; ncnn's and R-FCN Caffe's arithmetic) in fp32, every
 * operation rounded on its own (no FMA): input (batch, C, H, W) with C = output_dim * pooled_h * pooled_w, rois and item
 * layout as ROIPooling; output (batch * num_rois, output_dim, pooled_h, pooled_w).  For output (item, q, ph, pw):
 *   x1 = roundf(roi[0]) * spatial_scale, y1 likewise          (roundf: half away from zero)
 *   x2 = roundf(roi[2] + 1) * spatial_scale, y2 likewise with roi[3]
 *   roi_w = fmaxf(x2 - x1, 0.1), bin_w = roi_w / pooled_w     (roi_h, bin_h likewise)
 *   wstart = (int)floorf(x1 + pw * bin_w), wend = (int)ceilf(x1 + (pw + 1) * bin_w), converted saturating (NaN -> 0),
 *   then clamped to [0, W]                                    (h likewise)
 *   c = (q * pooled_h + ph) * pooled_w + pw
 *   value = 0 for an empty bin, else (the sum over the bin of plane c, row-major from 0) / (float)area: bit-exact.
 * Limits: -200 for pooled_h, pooled_w or output_dim < 1, spatial_scale not finite and > 0, or channels !=
 * output_dim * pooled_h * pooled_w; -100 for a NULL pointer or a size < 1.  Every RoI row is pooled, the [0, 0, 0, 0]
 * padding of fcuda_proposal_forward included. */
int fcuda_psroi_pooling_forward(float* output, const float* input, const float* rois, int channels, int height,
                                int width, int num_rois, int pooled_h, int pooled_w, int output_dim, float spatial_scale,
                                int batch, void* stream);

/* ---- Channel routing: ncnn's ShuffleChannel and Slice, and Concat -> ShuffleChannel -> Slice fused (the reference has
 * neither layer) ------------------------------------------------------------------------------------------------------
 * Every image of every blob is viewed as [outer][extent][inner].  The sources, concatenated along the middle axis, form
 * mid = sum of src_extent positions.  ShuffleChannel with k = reverse ? mid / group : group and cpg = mid / k puts
 * concatenated position cpg * i + j at shuffled position k * j + i (i < k, j < cpg); group 1 leaves the order alone.
 * Shuffled positions [dst_begin, dst_begin + sum of dst_extent) go to the destinations in order; the rest are not
 * written.  Each destination is (batch, outer, dst_extent[k], inner), each source (batch, outer, src_extent[k], inner).
 * Every output element is a bit copy of one input element; no input element is read twice.  One launch (one per 2^31
 * output elements of whole images), stream-ordered, nothing allocated: capturable in a CUDA graph.  16-byte accesses when
 * inner % 4 == 0 and every pointer is 16-byte aligned, 4-byte ones otherwise.
 * -100: a NULL route or pointer, batch < 1, outer, inner or an extent < 1, dst_begin < 0 or destinations past mid;
 * -200: num_src or num_dst outside 1..8, group < 1, mid % group != 0, or outer * inner * (sum of dst_extent) >= 2^31. */
#define FCUDA_ROUTE_MAX 8
typedef struct FcudaRoute {
    int outer, inner;
    int num_src;
    const float* src[FCUDA_ROUTE_MAX];
    int src_extent[FCUDA_ROUTE_MAX];
    int group, reverse;
    int dst_begin;
    int num_dst;
    float* dst[FCUDA_ROUTE_MAX];
    int dst_extent[FCUDA_ROUTE_MAX];
} FcudaRoute;
int fcuda_route_forward(const FcudaRoute* route, int batch, void* stream);
/* ncnn's Slice rule, host only.  A blob of ncnn rank `rank` (1..3) is stored as (c, h, w) = shape[0..2] (rank 2: c = 1;
 * rank 1: c = h = 1).  `axis` is the per-rank axis (rank 3: 0 = c, 1 = h, 2 = w; rank 2: 0 = h, 1 = w; rank 1: 0 = w; a
 * negative axis adds the rank); *storage_axis gets its index in (c, h, w).  Top i takes sizes[i] = slices[i], or for
 * slices[i] == -233 (extent - taken) / (count - i) where taken is what tops 0..i-1 took; the tops may leave a remainder.
 * -100: NULL pointers, count < 1, rank outside 1..3, a shape entry < 1; -200: the axis out of range, a size below 1, or
 * sizes past the extent. */
int fcuda_slice_plan(int rank, int axis, const int* shape, const int* slices, int count, int* storage_axis, int* sizes);

/* Kernel-variant switches for A/B measurements and tests.  Defaults are the measured-best configuration; the environment
 * variable FCUDA_<NAME> sets the initial value.  Names (value range, default):
 *   dw_vec (0-1, 1)           vectorised depthwise kernel on wide planes
 *   igemm_halo (0-1, 1)       implicit GEMM on stride-1, dense layers with IC % 32 == 0 (per group) and W % 4 == 0: the
 *                             input patch of 32 channels plus its halo arrives by one TMA load and serves every tap;
 *                             persistent CTAs, split and MMA of neighbouring k-blocks overlap.  0 = the gathering kernel
 *   igemm_presplit (0-1, 1)   halo kernel in fp32split mode: each 32-channel input box is split into its two bf16 planes
 *                             once instead of once per tap and the A fragments are loaded by ldmatrix (128-pixel
 *                             tiles).  Bit-identical to 0 = the per-tap split
 *   igemm_wide (0-1, 1)       read only when igemm_presplit is 1: the layers fcuda_igemm_wide_tile names run with the
 *                             GEMM turned around (output channels on the wgmma M side, 224 pixels per warpgroup on N,
 *                             read from the split planes by descriptor), so each filter byte serves 1.75x (N tile 128)
 *                             or 3.5x (N tile 64) as many pixels.  Bit-identical to 0 = the pre-split kernel
 *   igemm_stem (0-1, 1)       fp32split mode: the layers fcuda_igemm_stem_supported names (short K, e.g. IC = 3 first
 *                             layers) run on persistent CTAs that keep every filter k-block resident, gather the next
 *                             tile during the current one and write whole channel runs from a shared-memory staging
 *                             tile.  Bit-identical to 0 = the gathering kernel, one CTA per 128-pixel tile
 *   route_fuse (0-1, 1)       read by feather::Net's fusion pass when a net first fuses: Concat (axis 0) ->
 *                             ShuffleChannel -> Slice (axis 0) chains, or any two adjacent of them, run as one
 *                             fcuda_route_forward launch.  Bit-identical to 0 = every routing layer on its own, while
 *                             the net's other fusions stay as they are
 *   persistent_ctas (0-65536, 0)  n > 0: every persistent kernel (stem, halo / pre-split / wide implicit GEMM,
 *                             TensorGEMM) runs at most n CTAs, so each CTA walks ceil(tiles / n) or fewer tiles whatever
 *                             the card's SM count.  For tests; feather::Net captures grids in its CUDA graphs, so set it
 *                             before a Net first runs.  Bit-identical to 0 = as many CTAs as fit on the device
 * Every variant computes the same result (tests/test_gpu_variants.py).  Returns 0 / the value, -200 for an unknown name or value.
 * The retired names wino_mlp, gemm_pipe and yolo_nms are unknown names like any other: they return -200, and
 * FCUDA_WINO_MLP, FCUDA_GEMM_PIPE and FCUDA_YOLO_NMS are not read. */
int fcuda_set_tuning(const char* name, int value);
int fcuda_get_tuning(const char* name);

/* Profiling aid for bench.py's roofline leg: while enabled, every TensorGEMM launch is bracketed by CUDA events
 * on its own stream.  fcuda_profile_collect synchronises and reports, since the last enable: summed device time
 * (ms), the algorithmic FLOPs those launches stand for (direct-conv count, booster.h:145-148; 2*in*out*batch for
 * InnerProduct), the tensor-pipe FLOPs actually issued (x3 in TF32X3 mode) and the launch count. */
void fcuda_profile_tensor_gemm(int enable);
int fcuda_profile_collect(double* total_ms, double* algo_flops, double* mma_flops, long long* launches);
/* Same, per kernel class, for every instrumented launch (the enable switch above covers all of them):
 * kind 0 TensorGEMM, 1 implicit-GEMM conv, 2 Winograd input transform, 3 Winograd output transform, 4 pooling,
 * 5 depthwise, 6 element-wise (BN/Scale/Eltwise/BinaryOp/Clip/PReLU/Normalize/LRN), 7 deconvolution scatter / depthwise gather, 8 resize / crop (Interp,
 * Crop), 9 detection (Permute, axis Softmax, PriorBox, decode, NMS, merge; YOLO decode, select, mask, sweep), 10 channel
 * routing (fcuda_route_forward), 11 two-stage detection (Proposal decode, select, mask, sweep; ROIPooling; PSROIPooling),
 * 12 instance normalisation / padding (InstanceNorm, Padding), 13 pixel shuffle (PixelShuffle, alone or with its fused
 * upsampled-input add), 14 activation (Sigmoid, TanH, Swish, HardSigmoid, HardSwish, GELU), 15 attention
 * (fcuda_attention_forward), 16 layer normalisation (LayerNorm), < 0 all.  algo_bytes = the bytes the operation must move (inputs
 * read once + outputs written once). */
int fcuda_profile_collect_kind(int kind, double* total_ms, double* algo_flops, double* mma_flops, double* algo_bytes,
                               long long* launches);

/* Number of kernel launches issued by this library since the last reset (bench.py's gpu_launches). */
unsigned long long fcuda_launch_count(void);
void fcuda_reset_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FCUDA_H */
