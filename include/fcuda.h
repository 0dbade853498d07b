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

/* booster::ActivationType, booster.h:53-57 */
enum FcudaActivation { FCUDA_ACT_NONE = 0, FCUDA_ACT_RELU = 1 };

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
/* ReluLayer::Forward (src/layers/relu_layer.h:29-41). */
int fcuda_relu_forward(float* output, const float* input, size_t n, void* stream);
/* SoftmaxLayer::Forward (src/layers/softmax_layer.h:32-55): over each image's whole blob. */
int fcuda_softmax_forward(float* output, const float* input, size_t n_per_image, int batch, void* stream);
/* DropoutLayer::Forward (src/layers/dropout_layer.h:36-57): y = x*scale (copy when scale == 1). */
int fcuda_dropout_forward(float* output, const float* input, size_t n, float scale, void* stream);
/* ConcatLayer / SplitLayer copies (src/layers/concat_layer.h:37-47, split_layer.h:43-53): copies `channels`
 * channels of every image into dst at channel offset `dst_channel_offset` of a dst with `dst_channels`. */
int fcuda_copy_channels(float* dst, int dst_channels, int dst_channel_offset, const float* src, int channels,
                        size_t stride, int batch, void* stream);

/* Convolution with a fused Eltwise SUM (+ReLU): output = act(conv(input) [+bias] + residual), `residual` shaped like the
 * output.  Replaces ConvLayer::Forward followed by EltwiseLayer::Forward (src/layers/eltwise_layer.h:68-82 ->
 * booster::add_relu<>) when the Eltwise is the only reader of the convolution's top (ResNet shortcuts).  SGECONV adds the
 * residual in its epilogue; every other algorithm runs the convolution and then add_relu in place.  The convolution's
 * own activation (param->activation) is applied before the sum, relu_after_add after it. */
int fcuda_conv_forward_residual(const FcudaConvParam* param, int algo, float* output, const float* input,
                                const float* packed_kernel, float* scratch, const float* bias, const float* residual,
                                int relu_after_add, int batch, void* stream);

/* Convolution (+bias, +ReLU per param->activation) with a FOLLOWING 2x2 / stride-2 / pad-0 max pooling fused into its
 * epilogue (ConvLayer::Forward then PoolingLayer::Forward, src/layers/pooling_layer.h:38-91): `output` is the pooled blob
 * (batch, OC, (OH+1)/2, (OW+1)/2) — ceil mode, windows clipped at the border like the reference.  fcuda_conv_can_pool
 * says whether the algorithm can do it (Winograd F(6,3)/F(2,3): the output tile is pooled in registers; FCUDA_SGECONV:
 * 3x3 / stride-1 layers with IC % 32 == 0, pooled by two shuffles per value); otherwise the call returns -200. */
int fcuda_conv_can_pool(const FcudaConvParam* param, int algo);

/* FCUDA_SGECONV in the current arithmetic mode: 1 when the layer (output_h / output_w assigned) runs on the halo kernel
 * (switch igemm_halo below: stride 1, no dilation, more than one tap, input_channels / group % 32 == 0, input_w % 4 == 0,
 * 16-byte aligned input), with geom[0..3] = output patch rows, patch columns, shared-memory box rows, box columns;
 * 0 when it keeps the gathering kernel.  The switch itself is not consulted. */
int fcuda_igemm_halo_tile(const FcudaConvParam* param, int* geom);
/* The same for the pre-split halo kernel (switch igemm_presplit below; fp32split mode only): 1 when the layer runs on it,
 * with geom[0..3] = tile rows, tile columns (rows * columns = 256 where the layer's N tile is 64 output channels, else 128),
 * fp32 box rows, box columns; 0 otherwise.  The switch itself is not consulted. */
int fcuda_igemm_presplit_tile(const FcudaConvParam* param, int* geom);
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

/* Extended forward (beyond the reference, which rejects both: dilation at src/layers/conv_layer.h:43-47, partial groups at
 * avx/booster.cpp:304-308).  Same as fcuda_conv_forward[_residual] (`residual` may be NULL) plus a tap spacing.
 *   dilation: FCUDA_SGECONV only (-200 otherwise); the caller sets param->output_h/w for the dilated extent
 *             out = (in + pads - dilation*(k-1) - 1) / stride + 1.
 *   groups  : with FCUDA_SGECONV and param->group > 1 (also through the plain entry points) input_channels and
 *             output_channels are the TOTAL channel counts, the raw kernel is (OC, IC/group, KH, KW) and group g
 *             maps input channels [g*IC/G, (g+1)*IC/G) to output channels [g*OC/G, (g+1)*OC/G). */
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

/* Kernel-variant switches for A/B measurements and tests.  Defaults are the measured-best configuration; the environment
 * variable FCUDA_<NAME> sets the initial value.  Names (value range, default):
 *   dw_vec (0-1, 1)           vectorised depthwise kernel on wide planes
 *   wino_mlp (0-2, 2)         Winograd transforms: 1 = every global load of a block in flight at once (cp.async slab /
 *                             back-to-back plane loads) instead of register-staged rounds; 2 = also launch the channel
 *                             blocks of a tile group next to each other (whole 1 KB rows of V / M in flight together)
 *   igemm_halo (0-1, 1)       implicit GEMM on stride-1, dense layers with IC % 32 == 0 (per group) and W % 4 == 0: the
 *                             input patch of 32 channels plus its halo arrives by one TMA load and serves every tap;
 *                             persistent CTAs, split and MMA of neighbouring k-blocks overlap.  0 = the gathering kernel
 *   gemm_pipe (0-1, 1)        TensorGEMM (Winograd, im2col, InnerProduct): persistent CTAs that fill the next tile's ring
 *                             stages during the epilogue; the split and MMAs of neighbouring k-blocks overlap and no wgmma
 *                             waits for the one before it.  Bit-identical to 0 = one CTA per tile, drained per k-block
 *   igemm_presplit (0-1, 1)   halo kernel in fp32split mode: each 32-channel input box is split into its two bf16 planes
 *                             once instead of once per tap, the A fragments are loaded by ldmatrix, and layers with a
 *                             64-channel N tile use 256-pixel tiles.  Bit-identical to 0 = the per-tap split
 * Every variant computes the same result (tests/test_gpu_variants.py).  Returns 0 / the value, -200 for an unknown name or value. */
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
 * 5 depthwise, 6 element-wise (BN/Scale/Eltwise), 7 deconvolution scatter / depthwise gather, < 0 all.  algo_bytes = the bytes the operation must move (inputs
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
