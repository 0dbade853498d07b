// Clip and PReLU layers: ncnn's layer types of the same names (the reference has neither).  Clip is Caffe's ReLU6 with
// min 0 / max 6 and MobileNet-v2's activation; a Clip right after a convolution is folded into the convolution's epilogue
// by ConvLayer::Fuse, so this layer only runs when fusion is off or the Clip has no convolution producer.
#pragma once

#include <fcuda.h>
#include <feather/layer.h>
#include <float.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// y = min(max(x, min), max); 0 = min (default -FLT_MAX), 1 = max (default FLT_MAX).  NaN becomes min (see fcuda.h).
class ClipLayer : public Layer {
public:
    explicit ClipLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        min_value = pd.get(0, -FLT_MAX);
        max_value = pd.get(1, FLT_MAX);
        if (!(min_value <= max_value)) {
            LOGE("Clip layer %s: min %g is not <= max %g", this->name.c_str(), min_value, max_value);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Forward() {
        return fcuda_clip_forward(tops[0]->data(), bottoms[0]->data(), bottoms[0]->data_size(), min_value, max_value, stream());
    }
    float min_value = -FLT_MAX, max_value = FLT_MAX;
};

// y = x < 0 ? x * slope[c] : x; 0 = num_slope: one slope per channel, or 1 shared by all.  The slopes are the layer's
// only weight blob (num_slope floats in the model bin).
class PReLULayer : public Layer {
public:
    explicit PReLULayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        num_slope = pd.get(0, 0);
        if (num_slope <= 0) {
            LOGE("PReLU layer %s: num_slope %d", this->name.c_str(), num_slope);
            return FEATHER_ERR_WEIGHTS;
        }
        weights.push_back(NewWeightBlob(this->name + "_slope", 1, 1, 1, num_slope));
        return 0;
    }
    int LoadWeights(const ncnn::ModelBin& mb) {
        ncnn::Mat slope = mb.load(num_slope, 1);
        if (slope.empty() || weights.empty()) return FEATHER_ERR_WEIGHTS;
        return weights[0]->CopyDataFromMat(slope);
    }
    int Reshape() {
        const Blob<float>* b = bottoms[0];
        if (num_slope != 1 && static_cast<size_t>(num_slope) != b->channels()) {
            LOGE("PReLU layer %s has %d slopes for %zu channels", this->name.c_str(), num_slope, b->channels());
            return FEATHER_ERR_TOPOLOGY;
        }
        return Layer::Reshape();
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        return fcuda_prelu_forward(tops[0]->data(), b->data(), static_cast<int>(b->channels()), b->height() * b->width(),
                                   weights[0]->data(), num_slope, static_cast<int>(b->num()), stream());
    }

private:
    int num_slope = 0;
};

}  // inline namespace b200
}  // namespace feather
