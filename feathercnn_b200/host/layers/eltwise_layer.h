// EltwiseLayer (mirrors /root/reference/src/layers/eltwise_layer.h:21-90, which is SUM only without coefficients; PROD,
// MAX and SUM coefficients are this engine's extension, SURVEY.md §8f rank 4).
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

#include <vector>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class EltwiseLayer : public Layer {
public:
    explicit EltwiseLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param), op_type(1), fuse_relu(0) { _fusible = true; }

    int Reshape() {
        if (bottoms.size() < 2) return FEATHER_ERR_WEIGHTS;
        const size_t n = bottoms[0]->num(), c = bottoms[0]->channels(), h = bottoms[0]->height(), w = bottoms[0]->width();
        for (size_t i = 1; i < bottoms.size(); ++i)
            if (n != bottoms[i]->num() || c != bottoms[i]->channels() || h != bottoms[i]->height() || w != bottoms[i]->width()) {
                LOGE("Shape mismatch among bottoms of layer %s.", this->name.c_str());
                return FEATHER_ERR_WEIGHTS;
            }
        for (size_t i = 0; i < tops.size(); ++i) tops[i]->ReshapeWithRealloc(bottoms[0]);
        return 0;
    }

    // The reference accepts SUM without coefficients only (eltwise_layer.h:57-66); PROD / MAX / coefficients follow ncnn.
    int LoadParam(const ncnn::ParamDict& pd) {
        op_type = pd.get(0, 0);
        ncnn::Mat c = pd.get(1, ncnn::Mat());
        coeffs.clear();
        for (int i = 0; i < c.w; ++i) coeffs.push_back(c[i]);
        if (op_type < Operation_PROD || op_type > Operation_MAX) {
            LOGE("Eltwise layer %s: unknown operation %d", this->name.c_str(), op_type);
            return FEATHER_ERR_WEIGHTS;
        }
        if (!coeffs.empty() && op_type != Operation_SUM) return FEATHER_ERR_WEIGHTS;
        return 0;
    }

    bool plain_sum() const { return op_type == Operation_SUM && coeffs.empty(); }

    int Forward() {
        if (!coeffs.empty() && coeffs.size() != bottoms.size()) return FEATHER_ERR_WEIGHTS;
        const size_t n = bottoms[0]->data_size();
        if (plain_sum()) {
            // the reference adds bottoms 0 and 1 only (eltwise_layer.h:70-73); further bottoms are accumulated here
            int rc = fcuda_eltwise_add_forward(tops[0]->data(), bottoms[0]->data(), bottoms[1]->data(), n,
                                               (fuse_relu && bottoms.size() == 2) ? 1 : 0, stream());
            for (size_t i = 2; i < bottoms.size() && rc == 0; ++i)
                rc = fcuda_eltwise_add_forward(tops[0]->data(), tops[0]->data(), bottoms[i]->data(), n,
                                               (fuse_relu && i + 1 == bottoms.size()) ? 1 : 0, stream());
            return rc;
        }
        const float c0 = coeffs.empty() ? 1.f : coeffs[0], c1 = coeffs.empty() ? 1.f : coeffs[1];
        int rc = fcuda_eltwise_forward(tops[0]->data(), bottoms[0]->data(), bottoms[1]->data(), n, op_type, c0, c1,
                                       (fuse_relu && bottoms.size() == 2) ? 1 : 0, stream());
        for (size_t i = 2; i < bottoms.size() && rc == 0; ++i)
            rc = fcuda_eltwise_forward(tops[0]->data(), tops[0]->data(), bottoms[i]->data(), n, op_type, 1.f,
                                       coeffs.empty() ? 1.f : coeffs[i], (fuse_relu && i + 1 == bottoms.size()) ? 1 : 0,
                                       stream());
        return rc;
    }

    int Fuse(Layer* next_layer) {
        if (next_layer->type.compare("ReLU") == 0) {
            fuse_relu = 1;
            return 1;
        }
        return 0;
    }

    enum { Operation_PROD = 0, Operation_SUM = 1, Operation_MAX = 2 };
    int fused_relu() const { return fuse_relu; }

private:
    int op_type;
    int fuse_relu;
    std::vector<float> coeffs;
};

}  // inline namespace b200
}  // namespace feather
