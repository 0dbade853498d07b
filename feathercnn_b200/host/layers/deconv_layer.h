// DeconvLayer — serves ncnn "Deconvolution" and "DeconvolutionDepthWise" (transposed convolution; the reference has no
// such layer).  Same protocol as ConvLayer: LoadParam creates the weight / bias blobs, Reshape sizes the top and requests
// scratch, Init packs, Forward runs fcuda_deconv_forward.  Deliberately not a ConvLayer: Net::ApplyFusion's residual pass
// and LayerConvAlgo look for ConvLayer, and a deconvolution can fuse neither an Eltwise shortcut nor a pooling.  A
// following ReLU fuses (into the scatter / gather kernel) and a following Crop folds into the pads (FoldCrop);
// BatchNorm / Scale after it run as their own layers.
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

#include "resize_layers.h"

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class DeconvLayer : public Layer {
public:
    explicit DeconvLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {
        _fusible = true;
        param = FcudaDeconvParam();
    }
    ~DeconvLayer() { delete processed_weights; }

    int LoadParam(const ncnn::ParamDict& pd) {
        // ncnn's Deconvolution parameter ids
        param.output_channels = pd.get(0, 0);
        param.kernel_w = pd.get(1, 0);
        param.kernel_h = pd.get(11, param.kernel_w);
        param.dilation_w = pd.get(2, 1);
        param.dilation_h = pd.get(12, param.dilation_w);
        param.stride_w = pd.get(3, 1);
        param.stride_h = pd.get(13, param.stride_w);
        param.pad_left = pd.get(4, 0);
        param.pad_right = pd.get(15, param.pad_left);
        param.pad_top = pd.get(14, param.pad_left);
        param.pad_bottom = pd.get(16, param.pad_top);
        param.output_pad_right = pd.get(18, 0);
        param.output_pad_bottom = pd.get(19, param.output_pad_right);
        param.bias_term = pd.get(5, 0);
        param.group = pd.get(7, 1);
        param.activation = pd.get(9, 0);
        weight_data_size = pd.get(6, 0);
        if (pd.get(20, 0) || pd.get(21, 0)) {
            LOGE("Layer %s: output_w / output_h (ncnn \"same\" sizing) are not supported", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (pd.get(8, 0)) {
            LOGE("Layer %s: int8 deconvolution is not supported", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (param.pad_left < 0 || param.pad_right < 0 || param.pad_top < 0 || param.pad_bottom < 0 ||
            param.output_pad_right < 0 || param.output_pad_bottom < 0) {
            LOGE("Layer %s: negative (\"same\") padding is not supported", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (param.activation != FCUDA_ACT_NONE && param.activation != FCUDA_ACT_RELU) return FEATHER_ERR_UNSUPPORTED;
        if ((param.stride_h > 1 && param.dilation_h > 1) || (param.stride_w > 1 && param.dilation_w > 1))
            return FEATHER_ERR_UNSUPPORTED;
        if (param.group <= 0 || param.output_channels % param.group) return FEATHER_ERR_UNSUPPORTED;
        if (param.output_channels <= 0 || param.kernel_h <= 0 || param.kernel_w <= 0 || param.stride_h <= 0 ||
            param.stride_w <= 0 || param.dilation_h <= 0 || param.dilation_w <= 0)
            return FEATHER_ERR_WEIGHTS;
        const long long per_icg = static_cast<long long>(param.output_channels) * param.kernel_h * param.kernel_w;
        if (weight_data_size <= 0 || weight_data_size % per_icg) return FEATHER_ERR_WEIGHTS;
        const int icg = static_cast<int>(weight_data_size / per_icg);
        param.input_channels = icg * param.group;
        weights.push_back(NewWeightBlob(this->name + "_weights", param.output_channels, icg, param.kernel_h, param.kernel_w));
        if (param.bias_term) weights.push_back(NewWeightBlob(this->name + "_bias", param.output_channels, 1, 1, 1));
        return 0;
    }

    int LoadWeights(const ncnn::ModelBin& mb) {
        ncnn::Mat weight_data = mb.load(weight_data_size, 0);
        if (weight_data.empty() || this->weights.empty()) return FEATHER_ERR_WEIGHTS;
        int rc = this->weights[0]->CopyDataFromMat(weight_data);
        if (rc) return rc;
        if (param.bias_term) {
            ncnn::Mat bias_mat = mb.load(param.output_channels, 1);
            if (bias_mat.empty() || this->weights.size() < 2) return FEATHER_ERR_WEIGHTS;
            rc = weights[1]->CopyDataFromMat(bias_mat);
        }
        return rc;
    }

    int Reshape() {
        const Blob<float>* bottom = this->bottoms[0];
        if (param.input_channels != static_cast<int>(bottom->channels())) {
            LOGE("Loaded deconvolution layer %s has %d input channels while bottom blob has %zu channels",
                 this->name.c_str(), param.input_channels, bottom->channels());
            return FEATHER_ERR_TOPOLOGY;
        }
        param.input_h = bottom->height();
        param.input_w = bottom->width();
        if (crop_folded) {
            param.pad_top = own_pads[0]; param.pad_bottom = own_pads[1];
            param.pad_left = own_pads[2]; param.pad_right = own_pads[3];
        }
        int rc = fcuda_deconv_output_dim(&param);
        if (rc) return rc;
        if (crop_folded) {  // the folded Crop's window, from this input's (and the reference blob's) shape
            int oc = 0, oh = 0, ow = 0;
            if (!crop.Resolve(param.output_channels, param.output_h, param.output_w, crop_reference, &oc, &oh, &ow)) {
                LOGE("Layer %s: the folded crop window does not fit the %dx%d deconvolution output", this->name.c_str(),
                     param.output_h, param.output_w);
                return FEATHER_ERR_TOPOLOGY;
            }
            param.pad_top += crop.hoff;
            param.pad_left += crop.woff;
            param.pad_bottom += param.output_h - crop.hoff - oh;
            param.pad_right += param.output_w - crop.woff - ow;
            if ((rc = fcuda_deconv_output_dim(&param))) return rc;
        }
        const int batch = bottom->num();
        tops[0]->ReshapeWithRealloc(batch, param.output_channels, param.output_h, param.output_w);
        size_t scratch = 0, packed = 0;
        if ((rc = fcuda_deconv_get_buffer_size(&param, batch, &scratch, &packed))) return rc;
        MEMPOOL_CHECK_RETURN(this->common_mempool->Request(sizeof(float) * scratch));
        // the packed filter follows the equivalent convolution's algorithm, which the input size can change
        int algo = -1;
        if ((rc = fcuda_deconv_plan(&param, NULL, &algo))) return rc;
        if (init_algo >= 0 && init_algo != algo) return Init();
        return 0;
    }

    int Init() {
        size_t scratch = 0, packed = 0;
        int rc = fcuda_deconv_get_buffer_size(&param, 1, &scratch, &packed);
        if (rc) return rc;
        if (!processed_weights) processed_weights = new Blob<float>(this->name + "_proc_weights");
        processed_weights->ReshapeWithRealloc(1, 1, 1, static_cast<int>(packed));
        if (!processed_weights->data() || !weights[0]->data()) return FEATHER_ERR_WEIGHTS;
        if ((rc = fcuda_deconv_init(&param, processed_weights->data(), weights[0]->data(), stream()))) return rc;
        return fcuda_deconv_plan(&param, NULL, &init_algo);
    }

    int Forward() {
        float* buffer = NULL;
        MEMPOOL_CHECK_RETURN(this->common_mempool->GetPtr(&buffer));
        return fcuda_deconv_forward(&param, tops[0]->data(), bottoms[0]->data(), processed_weights->data(), buffer,
                                    param.bias_term ? weights[1]->data() : NULL, static_cast<int>(bottoms[0]->num()),
                                    stream());
    }

    int Fuse(Layer* next_layer) {
        if (param.activation != FCUDA_ACT_NONE || next_layer->type.compare("ReLU") != 0) return 0;
        param.activation = FCUDA_ACT_RELU;
        return 1;
    }

    // Net::ApplyFusion: a Crop of this layer's otherwise unread top, in h and w only, becomes part of the pads: pad_top
    // grows by hoff, pad_left by woff, pad_bottom / pad_right by what remains below and to the right of the window
    // (resolved in Reshape).  fcuda_deconv_forward crops by the pads on every path, so the result is bit-identical.  A
    // stride-1 layer that is not depthwise keeps its Crop: its plan depends on the pads (the direct convolution only while
    // every pad <= dilation * (K - 1)), and the grown pads are known only once the shapes are.  Returns 1 when folded.
    int FoldCrop(const CropWindow& window, Blob<float>* reference) {
        const bool depthwise = param.group > 1 && param.group == param.input_channels &&
                               param.output_channels == param.input_channels;
        if (crop_folded || window.coff != 0 || window.outc != 0) return 0;
        if (param.stride_h == 1 && param.stride_w == 1 && !depthwise) return 0;
        crop = window;
        crop_reference = reference;
        own_pads[0] = param.pad_top; own_pads[1] = param.pad_bottom;
        own_pads[2] = param.pad_left; own_pads[3] = param.pad_right;
        crop_folded = true;
        return 1;
    }

private:
    FcudaDeconvParam param;
    bool crop_folded = false;
    CropWindow crop;
    const Blob<float>* crop_reference = NULL;  // shape only; NULL for a one-bottom Crop
    int own_pads[4] = {0, 0, 0, 0};            // top, bottom, left, right as loaded
    int weight_data_size = 0;
    int init_algo = -1;
    Blob<float>* processed_weights = NULL;
};

}  // inline namespace b200
}  // namespace feather
