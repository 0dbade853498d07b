// LRNLayer: ncnn's LRN (the reference has none), the local response normalisation of AlexNet, CaffeNet and GoogLeNet
// (fcuda.h states the arithmetic).  It has no weights and takes part in no fusion.
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// 0 = region_type (0 ACROSS_CHANNELS, 1 WITHIN_CHANNEL), 1 = local_size (5), 2 = alpha (1), 3 = beta (0.75),
// 4 = bias (1, Caffe's k).
class LRNLayer : public Layer {
public:
    explicit LRNLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        region_type = pd.get(0, 0);
        local_size = pd.get(1, 5);
        alpha = pd.get(2, 1.f);
        beta = pd.get(3, 0.75f);
        bias = pd.get(4, 1.f);
        if (region_type < 0 || region_type > 1 || local_size < 1 || local_size % 2 == 0) {
            LOGE("LRN layer %s: region_type %d, local_size %d is not supported", this->name.c_str(), region_type,
                 local_size);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        return fcuda_lrn_forward(tops[0]->data(), b->data(), static_cast<int>(b->channels()), static_cast<int>(b->height()),
                                 static_cast<int>(b->width()), region_type, local_size, alpha, beta, bias,
                                 static_cast<int>(b->num()), stream());
    }

private:
    int region_type = 0, local_size = 5;
    float alpha = 1.f, beta = 0.75f, bias = 1.f;
};

}  // inline namespace b200
}  // namespace feather
