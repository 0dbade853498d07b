// ConvLayer — serves ncnn "Convolution" and "ConvolutionDepthWise" (mirrors
// /root/reference/src/layers/conv_layer.h:26-194; same ncnn param ids, same call protocol into ConvBooster).
#pragma once

#include <cuda_runtime_api.h>
#include <fcuda.h>
#include <feather/booster.h>
#include <feather/layer.h>
#include <stdlib.h>

#include <vector>

#include "clip_prelu_layers.h"
#include "pooling_layer.h"

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class ConvLayer : public Layer {
public:
    explicit ConvLayer(RuntimeParameter<float>* rt_param)
        : Layer(rt_param), bias_data(NULL), processed_kernel(NULL), processed_weights(NULL), init_algo(-1) {
        _fusible = true;
    }
    ~ConvLayer() {
        delete processed_weights;
        delete folded_bias;
        delete pre_pool;
    }

    int LoadParam(const ncnn::ParamDict& pd) {
        // The reference rejects dilation > 1 (conv_layer.h:41-47); here the implicit-GEMM and depthwise kernels space their taps
        dilation_w = pd.get(2, 1);
        dilation_h = pd.get(12, dilation_w);
        if (dilation_w < 1 || dilation_h < 1) return FEATHER_ERR_UNSUPPORTED;
        if (pd.get(8, 0)) {
            LOGE("int8 convolution is not supported in FeatherCNN.");
            return FEATHER_ERR_UNSUPPORTED;  // conv_layer.h:49-54
        }
        conv_param.kernel_w = pd.get(1, 0);
        conv_param.kernel_h = pd.get(11, conv_param.kernel_w);
        conv_param.stride_w = pd.get(3, 1);
        conv_param.stride_h = pd.get(13, conv_param.stride_w);
        conv_param.pad_left = pd.get(4, 0);
        conv_param.pad_bottom = pd.get(14, conv_param.pad_left);
        conv_param.pad_right = pd.get(4, 0);
        conv_param.pad_top = pd.get(14, conv_param.pad_left);
        conv_param.group = pd.get(7, 1);
        conv_param.output_channels = pd.get(0, 0);
        conv_param.bias_term = pd.get(5, 0);
        conv_param.activation = booster::None;
        const int weight_data_size = pd.get(6, 0);
        if (conv_param.group == 0 || conv_param.output_channels % conv_param.group) {
            LOGE("Layer %s output_channels is not divisible by its group", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;  // the reference exit(0)s here (conv_layer.h:70-74)
        }
        num_output = conv_param.output_channels;
        conv_param.output_channels /= conv_param.group;
        if (conv_param.output_channels <= 0 || conv_param.kernel_h <= 0 || conv_param.kernel_w <= 0) return FEATHER_ERR_WEIGHTS;
        conv_param.input_channels = weight_data_size / conv_param.output_channels / conv_param.kernel_h / conv_param.kernel_w;
        this->weight_data_size = weight_data_size;
        // Depthwise proper = one filter per channel.  `group == input_channels` alone (the reference's test, booster.h:121,
        // avx/booster.cpp:285) also matches an ordinary convolution over ONE input channel and truncates a depthwise
        // with a channel multiplier; those, and partial groups (rejected upstream, avx/booster.cpp:304-308), run as
        // grouped implicit GEMM with the TOTAL channel counts in conv_param.
        is_depthwise = conv_param.group > 1 && conv_param.group == conv_param.input_channels && num_output == conv_param.group;
        if (conv_param.group > 1 && !is_depthwise) {
            if (conv_param.input_channels % conv_param.group) return FEATHER_ERR_UNSUPPORTED;
            conv_param.output_channels = num_output;
            weights.push_back(NewWeightBlob(this->name + "_weights", num_output, conv_param.input_channels / conv_param.group,
                                            conv_param.kernel_h, conv_param.kernel_w));
        } else {
            weights.push_back(NewWeightBlob(this->name + "_weights", conv_param.output_channels, conv_param.input_channels,
                                            conv_param.kernel_h, conv_param.kernel_w));
        }
        if (conv_param.bias_term) {
            // The reference sizes the bias by output_channels/group (conv_layer.h:86), which is wrong for
            // depthwise-with-bias (SURVEY.md §8 quirks); the file holds num_output values, so read those.
            weights.push_back(NewWeightBlob(this->name + "_bias", num_output, 1, 1, 1));
        }
        return 0;
    }

    int LoadWeights(const ncnn::ModelBin& mb) {
        ncnn::Mat weight_data = mb.load(weight_data_size, 0);
        if (weight_data.empty() || this->weights.empty()) return FEATHER_ERR_WEIGHTS;
        int rc = this->weights[0]->CopyDataFromMat(weight_data);
        if (rc) return rc;
        if (conv_param.bias_term) {
            ncnn::Mat bias_mat = mb.load(num_output, 1);
            if (bias_mat.empty() || this->weights.size() < 2) return FEATHER_ERR_WEIGHTS;
            rc = weights[1]->CopyDataFromMat(bias_mat);
        }
        return rc;
    }

    int Reshape() {
        const Blob<float>* bottom_blob = this->bottoms[0];
        conv_param.input_w = bottom_blob->width();
        conv_param.input_h = bottom_blob->height();
        if (conv_param.input_channels != static_cast<int>(bottom_blob->channels())) {
            LOGE("Loaded convolution layer %s has %d input channels while bottom blob has %zu channels",
                 this->name.c_str(), conv_param.input_channels, bottom_blob->channels());
            return FEATHER_ERR_TOPOLOGY;
        }
        const int out_channels = is_depthwise ? conv_param.input_channels : num_output;
        conv_param.output_channels = out_channels;
        conv_param.AssignOutputDim();
        conv_param.output_channels = out_channels;  // AssignOutputDim applies the reference's group == IC rule (booster.h:121)
        if (dilation_h > 1 || dilation_w > 1) {
            conv_param.output_h = (conv_param.input_h + conv_param.pad_top + conv_param.pad_bottom -
                                   dilation_h * (conv_param.kernel_h - 1) - 1) / conv_param.stride_h + 1;
            conv_param.output_w = (conv_param.input_w + conv_param.pad_left + conv_param.pad_right -
                                   dilation_w * (conv_param.kernel_w - 1) - 1) / conv_param.stride_w + 1;
            if (conv_param.output_h <= 0 || conv_param.output_w <= 0) return FEATHER_ERR_WEIGHTS;
        }
        const int batch = bottom_blob->num();
        if (residual) {
            const int rc = CheckResidual(batch);
            if (rc) return rc;
        }
        if (fused_pool)  // the top is the pooled blob (ceil mode, pooling_layer.h:129-130 with k = s = 2, pad 0)
            tops[0]->ReshapeWithRealloc(batch, conv_param.output_channels, (conv_param.output_h + 1) / 2, (conv_param.output_w + 1) / 2);
        else
            tops[0]->ReshapeWithRealloc(batch, conv_param.output_channels, conv_param.output_h, conv_param.output_w);
        // FEATHER_ALGO_POLICY=reference keeps avx/booster.cpp:283-310 verbatim; default is the tuned cost model
        static const bool reference_policy = [] {
            const char* e = getenv("FEATHER_ALGO_POLICY");
            return e && e[0] == 'r';
        }();
        const bool extension = dilation_h > 1 || dilation_w > 1 || (conv_param.group > 1 && !is_depthwise) ||
                               (conv_param.group == 1 && conv_param.input_channels == 1);
        int rc = (reference_policy && !extension) ? conv_booster.SelectAlgo(&this->conv_param)
                                                  : conv_booster.SelectAlgoTuned(&this->conv_param);
        if (rc) return rc;
        if (dilation_h > 1 || dilation_w > 1)  // the depthwise kernels and the implicit GEMM space their taps
            conv_booster.ForceSelectAlgo(is_depthwise ? booster::DEPTHWISE : booster::SGECONV);
        if (const char* force = extension ? NULL : getenv("FEATHER_FORCE_CONV_ALGO")) {  // ForceSelectAlgo hook, avx/booster.cpp:313-317
            booster::ConvBooster forced;
            forced.ForceSelectAlgo(static_cast<booster::ConvAlgo>(atoi(force)));
            size_t a = 0, b = 0;
            if (conv_booster.GetAlgo() != booster::DEPTHWISE && forced.GetBufferSize(&conv_param, &a, &b, batch) == 0)
                conv_booster = forced;
        }
        size_t buffer_size = 0, dull = 0;
        rc = conv_booster.GetBufferSize(&conv_param, &buffer_size, &dull, batch);
        if (rc) return rc;
        MEMPOOL_CHECK_RETURN(this->common_mempool->Request(sizeof(float) * buffer_size));
        if (fused_pool) {
            // algorithms that cannot pool in their epilogue run the convolution into a private blob, then the pooling kernel
            pool_in_epilogue = dilation_h == 1 && dilation_w == 1 && fcuda_conv_can_pool(&conv_param, conv_booster.GetAlgo()) != 0;
            if (!pool_in_epilogue) {
                if (!pre_pool) pre_pool = new Blob<float>(this->name + "_pre_pool");
                pre_pool->ReshapeWithRealloc(batch, conv_param.output_channels, conv_param.output_h, conv_param.output_w);
                if (!pre_pool->data()) return FEATHER_ERR_CUDA;
            }
        }
        if (init_algo >= 0 && init_algo != conv_booster.GetAlgo()) return Init();  // shape change switched algorithms
        return 0;
    }

    int Init() {
        size_t buffer_size = 0, processed_kernel_size = 0;
        int rc = conv_booster.GetBufferSize(&conv_param, &buffer_size, &processed_kernel_size, 1);
        if (rc) return rc;
        if (!processed_weights) processed_weights = new Blob<float>(this->name + "_proc_weights");
        processed_weights->ReshapeWithRealloc(1, 1, 1, static_cast<int>(processed_kernel_size));
        if (!processed_weights->data() || !weights[0]->data()) return FEATHER_ERR_WEIGHTS;
        const float* raw = weights[0]->data();
        Blob<float> scaled_w(this->name + "_folded_weights");
        if (!fold_mul.empty()) {
            // BN/Scale folded into the filters: W'[oc] = W[oc] * mul[oc], b' = b * mul + add (exact algebra of
            // y = s*(beta*(conv + b) + alpha) + t; what the reference's dead Fuse hooks were meant to reach).
            const int oc = static_cast<int>(fold_mul.size());
            const size_t per_oc = weights[0]->data_size() / oc;
            Blob<float> mul_dev(this->name + "_fold_mul");
            mul_dev.ReshapeWithRealloc(1, 1, 1, oc);
            scaled_w.ReshapeWithRealloc(1, 1, 1, static_cast<int>(weights[0]->data_size()));
            if (!mul_dev.data() || !scaled_w.data()) return FEATHER_ERR_CUDA;
            if ((rc = mul_dev.CopyFromHost(fold_mul.data(), stream()))) return rc;
            rc = fcuda_scale_forward(scaled_w.data(), raw, oc, per_oc, mul_dev.data(), NULL, 1, stream());
            if (rc) return rc;
            std::vector<float> b(oc, 0.f);
            if (had_bias) {
                if ((rc = weights[1]->CopyToHost(b.data(), stream()))) return rc;
            }
            for (int i = 0; i < oc; ++i) b[i] = b[i] * fold_mul[i] + fold_add[i];
            if (!folded_bias) folded_bias = new Blob<float>(this->name + "_folded_bias");
            folded_bias->ReshapeWithRealloc(1, 1, 1, oc);
            if (!folded_bias->data()) return FEATHER_ERR_CUDA;
            if ((rc = folded_bias->CopyFromHost(b.data(), stream()))) return rc;
            raw = scaled_w.data();
        }
        rc = conv_booster.Init(&conv_param, processed_weights->data(), raw, stream());
        if (rc) return rc;
        if (!fold_mul.empty()) {
            // scaled_w / mul_dev are released when this scope ends: make sure the kernels reading them finished
            if (cudaStreamSynchronize(static_cast<cudaStream_t>(stream())) != cudaSuccess) return FEATHER_ERR_CUDA;
        }
        this->processed_kernel = processed_weights->data();
        if (!fold_mul.empty()) bias_data = folded_bias->data();
        else if (conv_param.bias_term) bias_data = this->weights[1]->data();
        init_algo = conv_booster.GetAlgo();
        return 0;
    }

    int Forward() {
        float* buffer = NULL;
        MEMPOOL_CHECK_RETURN(this->common_mempool->GetPtr(&buffer));
        const int batch = static_cast<int>(bottoms[0]->num());
        FcudaConvOptions o = FcudaConvOptions();
        o.residual = residual && !residual_broadcast ? residual->data() : NULL;
        o.relu_after_add = relu_after_add;
        o.clip_min = clip_min; o.clip_max = clip_max;
        o.dilation_h = dilation_h; o.dilation_w = dilation_w;
        o.pool = fused_pool && pool_in_epilogue;
        const bool pool_after = fused_pool && !pool_in_epilogue;
        const int rc = conv_booster.ForwardOpts(&conv_param, pool_after ? pre_pool->data() : tops[0]->data(), bottoms[0]->data(),
                                                processed_kernel, buffer, bias_data, o, batch, stream());
        if (!rc && residual_broadcast) {  // a broadcast addend: the BinaryOp ADD (+ReLU) in place after the convolution
            const int out[4] = {batch, conv_param.output_channels, conv_param.output_h, conv_param.output_w};
            return fcuda_binary_op_forward(tops[0]->data(), tops[0]->data(), out, residual->data(), residual_shape, 0.f,
                                           FCUDA_BINARY_ADD, relu_after_add, stream());
        }
        if (rc || !pool_after) return rc;
        return fcuda_pooling_forward(tops[0]->data(), pre_pool->data(), conv_param.output_channels, conv_param.output_h,
                                     conv_param.output_w, 0, 2, 2, 2, 2, 0, 0, 0, 0, 0, batch, stream());
    }

    // Net::ApplyFusion: absorb `Eltwise SUM(this->top, other) [+ReLU]` (a ResNet shortcut), or the same add written as a
    // BinaryOp ADD (`broadcast`: `other` may broadcast against this layer's output), into this layer's epilogue.
    int FuseResidual(Blob<float>* other, int relu, bool broadcast) {
        if (residual != NULL || fused_pool || (is_depthwise && (dilation_h > 1 || dilation_w > 1))) return 0;
        residual = other;
        relu_after_add = relu;
        residual_may_broadcast = broadcast;
        return 1;
    }

    // Reshape with a fused residual, whose shape is only known now: an addend shaped like the output goes to the
    // epilogue; a BinaryOp addend that broadcasts onto the output (fcuda_binary_op_shape, the output on the left) is
    // added after the convolution by fcuda_binary_op_forward; anything else is the topology error the unfused layer
    // would report.
    int CheckResidual(int batch) {
        const int oc = conv_param.output_channels, oh = conv_param.output_h, ow = conv_param.output_w;
        const Blob<float>* r = residual;
        residual_broadcast = false;
        if (r->num() == static_cast<size_t>(batch) && r->channels() == static_cast<size_t>(oc) &&
            r->height() == static_cast<size_t>(oh) && r->width() == static_cast<size_t>(ow))
            return 0;
        const int mine[3] = {oc, oh, ow};
        const int theirs[3] = {static_cast<int>(r->channels()), static_cast<int>(r->height()), static_cast<int>(r->width())};
        int rank = 0, out[3], a[3];
        if (residual_may_broadcast && r->num() == static_cast<size_t>(batch) &&
            fcuda_binary_op_shape(3, mine, r->dims(), theirs, &rank, out, a, residual_shape + 1) == 0 && rank == 3 &&
            out[0] == oc && out[1] == oh && out[2] == ow) {
            residual_shape[0] = batch;
            residual_broadcast = true;
            return 0;
        }
        LOGE("Convolution layer %s: the added blob %s (%zu, %zu, %zu, %zu) does not fit its output (%d, %d, %d, %d)",
             this->name.c_str(), r->name.c_str(), r->num(), r->channels(), r->height(), r->width(), batch, oc, oh, ow);
        return FEATHER_ERR_TOPOLOGY;
    }

    // conv_layer.h:174-185, extended to BatchNorm, Scale, Clip and a trailing 2x2 max pooling
    int Fuse(Layer* next_layer) {
        if (fused_pool) return 0;  // the pooling is always last
        if (next_layer->type.compare("Pooling") == 0) {
            PoolingLayer* pl = dynamic_cast<PoolingLayer*>(next_layer);
            // A clamped convolution keeps its pooling separate: a Clip followed by the pooling in one epilogue is not built.
            if (!pl || !pl->IsMax2x2Stride2() || residual != NULL || conv_param.activation == booster::Clip) return 0;
            fused_pool = true;
            return 1;
        }
        if (conv_param.activation != booster::None) return 0;  // the activation precedes only the pooling
        if (next_layer->type.compare("ReLU") == 0) {
            conv_param.activation = booster::ReLU;
            return 1;
        }
        if (next_layer->type.compare("Clip") == 0) {
            // after any BatchNorm / Scale folding, so conv -> BN -> Scale -> Clip is one kernel.  A Clip in the epilogue of a
            // dilated ordinary convolution, or before a residual sum, is not built: there the Clip stays a layer of its own.
            // A dilated depthwise layer clamps in its epilogue like an undilated one.
            const ClipLayer* cl = dynamic_cast<const ClipLayer*>(next_layer);
            if (!cl || residual != NULL || (!is_depthwise && (dilation_h > 1 || dilation_w > 1))) return 0;
            conv_param.activation = booster::Clip;
            clip_min = cl->min_value;
            clip_max = cl->max_value;
            return 1;
        }
        const bool is_bn = next_layer->type.compare("BatchNorm") == 0;
        const bool is_scale = next_layer->type.compare("Scale") == 0;
        if (!is_bn && !is_scale) return 0;
        if (next_layer->weights.empty() || !next_layer->weights[0]->data()) return 0;
        const int oc = static_cast<int>(next_layer->weights[0]->data_size());
        if (oc != num_output) return 0;
        std::vector<float> m(oc, 1.f), a(oc, 0.f);
        if (is_bn) {  // weights = {alpha, beta}: y = beta*x + alpha (batchnorm_layer.h:70-75)
            if (next_layer->weights.size() < 2 || !next_layer->weights[1]->data()) return 0;
            if (next_layer->weights[0]->CopyToHost(a.data(), stream()) || next_layer->weights[1]->CopyToHost(m.data(), stream())) return 0;
        } else {      // weights = {scale[, bias]}: y = x*scale + bias (scale_layer.h:75-86)
            if (next_layer->weights[0]->CopyToHost(m.data(), stream())) return 0;
            if (next_layer->weights.size() > 1 && next_layer->weights[1]->CopyToHost(a.data(), stream())) return 0;
        }
        if (fold_mul.empty()) {
            fold_mul.assign(oc, 1.f);
            fold_add.assign(oc, 0.f);
            had_bias = conv_param.bias_term != 0;
            conv_param.bias_term = 1;
        }
        for (int i = 0; i < oc; ++i) {
            fold_add[i] = fold_add[i] * m[i] + a[i];
            fold_mul[i] = fold_mul[i] * m[i];
        }
        return 1;
    }

    const booster::ConvParam& param() const { return conv_param; }
    int algo() const { return conv_booster.GetAlgo(); }

protected:
    booster::ConvBooster conv_booster;
    booster::ConvParam conv_param;
    float* bias_data;
    float* processed_kernel;
    Blob<float>* processed_weights;
    int init_algo;
    int num_output = 0;
    int weight_data_size = 0;
    int dilation_h = 1, dilation_w = 1;
    bool is_depthwise = false;
    // BN / Scale folding (Net::SetFusion): per-output-channel multiplier and offset applied at Init
    std::vector<float> fold_mul, fold_add;
    bool had_bias = false;
    Blob<float>* folded_bias = NULL;
    // fused Clip (ConvLayer::Fuse): the epilogue's clamp bounds when conv_param.activation == booster::Clip
    float clip_min = 0.f, clip_max = 0.f;
    // fused Eltwise SUM or BinaryOp ADD (Net::ApplyFusion); a BinaryOp addend may broadcast, and when it does
    // (CheckResidual) residual_shape holds its (n, c, h, w) along the output's axes
    Blob<float>* residual = NULL;
    int relu_after_add = 0;
    bool residual_may_broadcast = false, residual_broadcast = false;
    int residual_shape[4] = {0, 0, 0, 0};
    // fused trailing 2x2 / stride-2 max pooling (Net::ApplyFusion)
    bool fused_pool = false;
    bool pool_in_epilogue = false;
    Blob<float>* pre_pool = NULL;

};

}  // inline namespace b200
}  // namespace feather
