// InstanceNormLayer and PaddingLayer: ncnn's InstanceNorm and Padding, the layers of fast neural style transfer
// (Johnson et al.'s transformer network; the reference has neither).  InstanceNorm absorbs a following ReLU and then a
// following Padding into its write (fcuda_instance_norm_forward), so IN -> ReLU -> Padding is one pass over the plane
// after the statistics; Padding never fuses on its own.
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// 0 = top, 1 = bottom, 2 = left, 3 = right (0), 4 = type (0 constant, 1 replicate, 2 reflect), 5 = value (0.f);
// 6 = per_channel_pad_data_size, 7 = front, 8 = behind must be 0.  No weights.
class PaddingLayer : public Layer {
public:
    explicit PaddingLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        pad.top = pd.get(0, 0);
        pad.bottom = pd.get(1, 0);
        pad.left = pd.get(2, 0);
        pad.right = pd.get(3, 0);
        pad.type = pd.get(4, 0);
        pad.value = pd.get(5, 0.f);
        const int per_channel = pd.get(6, 0), front = pd.get(7, 0), behind = pd.get(8, 0);
        if (per_channel || front || behind || pad.top < 0 || pad.bottom < 0 || pad.left < 0 || pad.right < 0 ||
            pad.type < 0 || pad.type > 2) {
            LOGE("Padding layer %s: pads %d %d %d %d, type %d, per_channel_pad_data_size %d, front %d, behind %d is not "
                 "supported", this->name.c_str(), pad.top, pad.bottom, pad.left, pad.right, pad.type, per_channel, front,
                 behind);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() { return ReshapePadded(this, pad); }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        return fcuda_padding_forward(tops[0]->data(), b->data(), static_cast<int>(b->channels()),
                                     static_cast<int>(b->height()), static_cast<int>(b->width()), &pad,
                                     static_cast<int>(b->num()), stream());
    }
    const FcudaPad& param() const { return pad; }

    // Shapes `layer`'s top as its bottom padded by `p`; FEATHER_ERR_TOPOLOGY for a reflect pad >= the dimension it pads.
    static int ReshapePadded(Layer* layer, const FcudaPad& p) {
        const Blob<float>* b = layer->bottoms[0];
        const size_t h = b->height(), w = b->width();
        if (p.type == 2 && (static_cast<size_t>(p.top) >= h || static_cast<size_t>(p.bottom) >= h ||
                            static_cast<size_t>(p.left) >= w || static_cast<size_t>(p.right) >= w)) {
            LOGE("Layer %s: reflect pads %d %d %d %d on a %zu x %zu plane", layer->name.c_str(), p.top, p.bottom, p.left,
                 p.right, h, w);
            return FEATHER_ERR_TOPOLOGY;
        }
        layer->tops[0]->ReshapeWithRealloc(b->num(), b->channels(), h + p.top + p.bottom, w + p.left + p.right);
        return 0;
    }

private:
    FcudaPad pad = FcudaPad();
};

// 0 = channels, 1 = eps (0.001), 2 = affine (1): with affine the weights are gamma then beta, `channels` raw floats
// each.  The statistics' workspace comes from the common pool.
class InstanceNormLayer : public Layer {
public:
    explicit InstanceNormLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) { _fusible = true; }
    int LoadParam(const ncnn::ParamDict& pd) {
        channels = pd.get(0, 0);
        eps = pd.get(1, 0.001f);
        affine = pd.get(2, 1);
        if (channels < 1 || !(eps >= 0.f)) {
            LOGE("InstanceNorm layer %s: channels %d, eps %g is not supported", this->name.c_str(), channels, eps);
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (affine) {
            weights.push_back(NewWeightBlob(this->name + "_gamma", 1, 1, 1, channels));
            weights.push_back(NewWeightBlob(this->name + "_beta", 1, 1, 1, channels));
        }
        return 0;
    }
    int LoadWeights(const ncnn::ModelBin& mb) {
        if (!affine) return 0;
        ncnn::Mat gamma = mb.load(channels, 1);
        ncnn::Mat beta = mb.load(channels, 1);
        if (gamma.empty() || beta.empty() || weights.size() != 2) return FEATHER_ERR_WEIGHTS;
        const int rc = weights[0]->CopyDataFromMat(gamma);
        return rc ? rc : weights[1]->CopyDataFromMat(beta);
    }
    // A ReLU (its slope ignored, as ReluLayer does), then a Padding, which is always last.
    int Fuse(Layer* next_layer) {
        if (fuse_pad) return 0;
        if (next_layer->type == "ReLU" && !fuse_relu) {
            fuse_relu = true;
            return 1;
        }
        PaddingLayer* p = dynamic_cast<PaddingLayer*>(next_layer);
        if (p) {
            fuse_pad = true;
            pad = p->param();
            return 1;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* b = bottoms[0];
        if (static_cast<size_t>(channels) != b->channels()) {
            LOGE("InstanceNorm layer %s has %d channels, its bottom %zu", this->name.c_str(), channels, b->channels());
            return FEATHER_ERR_TOPOLOGY;
        }
        size_t floats = 0;
        const int rc = fcuda_instance_norm_workspace_size(channels, b->height() * b->width(), static_cast<int>(b->num()),
                                                          &floats);
        if (rc) return rc;
        if (!this->common_mempool->Request(sizeof(float) * floats)) return FEATHER_ERR_CUDA;
        return PaddingLayer::ReshapePadded(this, pad);
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        float* workspace = NULL;
        if (!this->common_mempool->GetPtr(&workspace)) return FEATHER_ERR_CUDA;
        return fcuda_instance_norm_forward(tops[0]->data(), b->data(), channels, static_cast<int>(b->height()),
                                           static_cast<int>(b->width()), affine ? weights[0]->data() : NULL,
                                           affine ? weights[1]->data() : NULL, eps, fuse_relu ? 1 : 0,
                                           fuse_pad ? &pad : NULL, workspace, static_cast<int>(b->num()), stream());
    }

private:
    int channels = 0, affine = 1;
    float eps = 0.001f;
    bool fuse_relu = false, fuse_pad = false;
    FcudaPad pad = FcudaPad();  // all zero: no padding
};

}  // inline namespace b200
}  // namespace feather
