// ActivationLayer: ncnn's Sigmoid, TanH, Swish, HardSigmoid, HardSwish and GELU (the reference has none), one class for
// the six type names.  MobileNet-v3 uses HardSwish and HardSigmoid (its squeeze-and-excitation gate), EfficientNet Swish
// and Sigmoid, ESPCN TanH, Vision Transformers GELU.  Each runs as its own element-wise pass over the whole blob, of any rank: no layer folds into
// a convolution or absorbs one (_fusible stays false, and ConvLayer::Fuse takes none of them).
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

#include <math.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// HardSigmoid / HardSwish: 0 = alpha (0.2), 1 = beta (0.5); GELU: 0 = fast_gelu (0 erf, 1 tanh); the other three
// take no parameters.  No weights.
class ActivationLayer : public Layer {
public:
    explicit ActivationLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        if (!type.compare("Sigmoid")) act = FCUDA_ACTIVATION_SIGMOID;
        else if (!type.compare("TanH")) act = FCUDA_ACTIVATION_TANH;
        else if (!type.compare("Swish")) act = FCUDA_ACTIVATION_SWISH;
        else if (!type.compare("HardSigmoid")) act = FCUDA_ACTIVATION_HARDSIGMOID;
        else if (!type.compare("HardSwish")) act = FCUDA_ACTIVATION_HARDSWISH;
        else if (!type.compare("GELU")) {
            const int fast = pd.get(0, 0);
            if (fast != 0 && fast != 1) {
                LOGE("GELU layer %s: fast_gelu %d is not supported (0 or 1)", this->name.c_str(), fast);
                return FEATHER_ERR_UNSUPPORTED;
            }
            act = fast ? FCUDA_ACTIVATION_GELU_TANH : FCUDA_ACTIVATION_GELU;
        } else return FEATHER_ERR_UNSUPPORTED;
        const bool hard = act == FCUDA_ACTIVATION_HARDSIGMOID || act == FCUDA_ACTIVATION_HARDSWISH;
        if (hard) {
            alpha = pd.get(0, 0.2f);
            beta = pd.get(1, 0.5f);
        }
        if (bottoms.size() != 1 || tops.size() != 1 || (hard && (alpha == 0.f || !isfinite(alpha) || !isfinite(beta)))) {
            LOGE("%s layer %s: alpha %g, beta %g with %zu bottoms and %zu tops is not supported (alpha finite and not 0, "
                 "beta finite; one bottom, one top)", type.c_str(), this->name.c_str(), alpha, beta, bottoms.size(),
                 tops.size());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Forward() {
        return fcuda_activation_forward(tops[0]->data(), bottoms[0]->data(), bottoms[0]->data_size(), act, alpha, beta,
                                        stream());
    }

private:
    int act = FCUDA_ACTIVATION_SIGMOID;
    float alpha = 0.2f, beta = 0.5f;
};

}  // inline namespace b200
}  // namespace feather
