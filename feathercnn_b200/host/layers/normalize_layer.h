// NormalizeLayer: ncnn's Normalize (the reference has none), weiliu89's SSD conv4_3_norm: an L2 normalisation of each
// pixel across its channels, of each channel plane or of the whole image, then a learned scale (fcuda.h states the
// arithmetic).  It takes part in no fusion.
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// 0 = across_spatial (0), 1 = channel_shared (0), 2 = eps (1e-4), 3 = scale_data_size, 4 = across_channel (1),
// 9 = eps_mode (0).  The scales are the layer's only weight blob: scale_data_size raw floats in the model bin.
class NormalizeLayer : public Layer {
public:
    explicit NormalizeLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        across_spatial = pd.get(0, 0);
        channel_shared = pd.get(1, 0);
        eps = pd.get(2, 0.0001f);
        scale_data_size = pd.get(3, 0);
        across_channel = pd.get(4, 1);
        eps_mode = pd.get(9, 0);
        if (scale_data_size < 1) {
            LOGE("Normalize layer %s: scale_data_size %d", this->name.c_str(), scale_data_size);
            return FEATHER_ERR_WEIGHTS;
        }
        if (eps_mode < 0 || eps_mode > 2 || (!across_spatial && !across_channel) || !(eps >= 0.f)) {
            LOGE("Normalize layer %s: across_spatial %d, across_channel %d, eps %g, eps_mode %d is not supported",
                 this->name.c_str(), across_spatial, across_channel, eps, eps_mode);
            return FEATHER_ERR_UNSUPPORTED;
        }
        weights.push_back(NewWeightBlob(this->name + "_scale", 1, 1, 1, scale_data_size));
        return 0;
    }
    int LoadWeights(const ncnn::ModelBin& mb) {
        ncnn::Mat scale = mb.load(scale_data_size, 1);
        if (scale.empty() || weights.empty()) return FEATHER_ERR_WEIGHTS;
        return weights[0]->CopyDataFromMat(scale);
    }
    // Top shaped like the bottom (its ncnn rank too); the across_spatial modes size their workspace in the common pool.
    int Reshape() {
        const Blob<float>* b = bottoms[0];
        if (!channel_shared && static_cast<size_t>(scale_data_size) != b->channels()) {
            LOGE("Normalize layer %s has %d scales for %zu channels", this->name.c_str(), scale_data_size, b->channels());
            return FEATHER_ERR_TOPOLOGY;
        }
        size_t floats = 0;
        const int rc = fcuda_normalize_workspace_size(across_spatial, across_channel, static_cast<int>(b->channels()),
                                                      b->height() * b->width(), static_cast<int>(b->num()), &floats);
        if (rc) return rc;
        if (floats && !this->common_mempool->Request(sizeof(float) * floats)) return FEATHER_ERR_CUDA;
        return Layer::Reshape();
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        float* workspace = NULL;
        if (across_spatial && !this->common_mempool->GetPtr(&workspace)) return FEATHER_ERR_CUDA;
        // a channel_shared layer reads scale[0] whatever scale_data_size is, as ncnn does
        return fcuda_normalize_forward(tops[0]->data(), b->data(), static_cast<int>(b->channels()), b->height() * b->width(),
                                       weights[0]->data(), channel_shared ? 1 : scale_data_size, across_spatial,
                                       across_channel, eps, eps_mode, workspace, static_cast<int>(b->num()), stream());
    }

private:
    int across_spatial = 0, channel_shared = 0, scale_data_size = 0, across_channel = 1, eps_mode = 0;
    float eps = 0.0001f;
};

}  // inline namespace b200
}  // namespace feather
