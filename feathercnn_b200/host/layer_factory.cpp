// Built-in layer registrations: the 13 ncnn type names the reference serves (/root/reference/src/layer_factory.cpp:53-68)
// plus Deconvolution / DeconvolutionDepthWise, Interp, Crop, Clip, PReLU, SSD's Permute, Flatten, Reshape, PriorBox and
// DetectionOutput, VGG-SSD's Normalize, YOLO's YoloDetectionOutput and Yolov3DetectionOutput, ShuffleNet's ShuffleChannel
// and Slice, AlexNet's and GoogLeNet's LRN, Faster R-CNN's Proposal and ROIPooling, R-FCN's PSROIPooling, fast neural
// style's InstanceNorm and Padding, super-resolution's PixelShuffle, BinaryOp (the element-wise ops onnx2ncnn and pnnx
// write, residual adds among them), the activations Sigmoid, TanH, Swish, HardSigmoid and HardSwish (MobileNet-v3,
// EfficientNet, ESPCN), and Vision Transformers' GELU, LayerNorm, MemoryData and MultiHeadAttention, 46 in all, mapped
// onto this host's layer classes.  A table of {type name,
// factory} pairs instead of one macro line per layer; the
// DEFINE_LAYER_CREATOR / REGISTER_LAYER_CREATOR macros of <feather/layer_factory.h> remain the plugin API for user layers.
#include <feather/layer_factory.h>

#include <stdio.h>

#include "layers/activation_layers.h"
#include "layers/batchnorm_layer.h"
#include "layers/binary_op_layer.h"
#include "layers/clip_prelu_layers.h"
#include "layers/conv_layer.h"
#include "layers/deconv_layer.h"
#include "layers/detection_layers.h"
#include "layers/eltwise_layer.h"
#include "layers/inner_product_layer.h"
#include "layers/lrn_layer.h"
#include "layers/misc_layers.h"
#include "layers/normalize_layer.h"
#include "layers/pixel_shuffle_layer.h"
#include "layers/pooling_layer.h"
#include "layers/rcnn_layers.h"
#include "layers/relu_layer.h"
#include "layers/resize_layers.h"
#include "layers/route_layers.h"
#include "layers/scale_layer.h"
#include "layers/style_layers.h"
#include "layers/transformer_layers.h"
#include "layers/yolo_layers.h"

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

namespace {

template <class L>
Layer* make_layer(RuntimeParameter<float>* rt_param) {
    return new L(rt_param);
}

struct BuiltIn {
    const char* ncnn_type;
    LayerRegistry::Creator create;
};

// "Convolution" and "ConvolutionDepthWise" share one class: group == channels selects the depthwise algorithm; so do
// "Deconvolution" and "DeconvolutionDepthWise".
const BuiltIn kBuiltIns[] = {
    {"Input", make_layer<InputLayer>},
    {"Convolution", make_layer<ConvLayer>},
    {"ConvolutionDepthWise", make_layer<ConvLayer>},
    {"InnerProduct", make_layer<InnerProductLayer>},
    {"Pooling", make_layer<PoolingLayer>},
    {"BatchNorm", make_layer<BatchNormLayer>},
    {"Scale", make_layer<ScaleLayer>},
    {"Eltwise", make_layer<EltwiseLayer>},
    {"ReLU", make_layer<ReluLayer>},
    {"Softmax", make_layer<SoftmaxLayer>},
    {"Dropout", make_layer<DropoutLayer>},
    {"Split", make_layer<SplitLayer>},
    {"Concat", make_layer<ConcatLayer>},
    {"Deconvolution", make_layer<DeconvLayer>},
    {"DeconvolutionDepthWise", make_layer<DeconvLayer>},
    {"Interp", make_layer<InterpLayer>},
    {"Crop", make_layer<CropLayer>},
    {"Clip", make_layer<ClipLayer>},
    {"PReLU", make_layer<PReLULayer>},
    {"Permute", make_layer<PermuteLayer>},
    {"Flatten", make_layer<FlattenLayer>},
    {"Reshape", make_layer<ReshapeLayer>},
    {"PriorBox", make_layer<PriorBoxLayer>},
    {"DetectionOutput", make_layer<DetectionOutputLayer>},
    {"Normalize", make_layer<NormalizeLayer>},
    {"YoloDetectionOutput", make_layer<YoloDetectionOutputLayer>},
    {"Yolov3DetectionOutput", make_layer<Yolov3DetectionOutputLayer>},
    {"ShuffleChannel", make_layer<ShuffleChannelLayer>},
    {"Slice", make_layer<SliceLayer>},
    {"LRN", make_layer<LRNLayer>},
    {"Proposal", make_layer<ProposalLayer>},
    {"ROIPooling", make_layer<ROIPoolingLayer>},
    {"PSROIPooling", make_layer<PSROIPoolingLayer>},
    {"InstanceNorm", make_layer<InstanceNormLayer>},
    {"Padding", make_layer<PaddingLayer>},
    {"PixelShuffle", make_layer<PixelShuffleLayer>},
    {"BinaryOp", make_layer<BinaryOpLayer>},
    {"Sigmoid", make_layer<ActivationLayer>},
    {"TanH", make_layer<ActivationLayer>},
    {"Swish", make_layer<ActivationLayer>},
    {"HardSigmoid", make_layer<ActivationLayer>},
    {"HardSwish", make_layer<ActivationLayer>},
    {"GELU", make_layer<ActivationLayer>},
    {"LayerNorm", make_layer<LayerNormLayer>},
    {"MemoryData", make_layer<MemoryDataLayer>},
    {"MultiHeadAttention", make_layer<MultiHeadAttentionLayer>},
};

}  // namespace

LayerRegistry::CreatorRegistry& LayerRegistry::Registry() {
    static CreatorRegistry* table = new CreatorRegistry();  // never destroyed: layers may be created during exit
    return *table;
}

void LayerRegistry::AddCreator(const std::string& type, Creator creator) { Registry()[type] = creator; }

Layer* LayerRegistry::CreateLayer(std::string type, RuntimeParameter<float>* rt_param) {
    const CreatorRegistry& table = Registry();
    const CreatorRegistry::const_iterator hit = table.find(type);
    if (hit == table.end()) {
        fprintf(stderr, "Layer type %s is not supported in FeatherCNN...Aborting\n", type.c_str());
        return NULL;
    }
    return hit->second(rt_param);
}

void register_layer_creators() {
    for (const BuiltIn& b : kBuiltIns) LayerRegistry::AddCreator(b.ncnn_type, b.create);
}

}  // inline namespace b200
}  // namespace feather
