// PermuteLayer, FlattenLayer, ReshapeLayer, PriorBoxLayer and DetectionOutputLayer — ncnn's layers of those names, the
// head of single-shot detectors (MobileNet-SSD, VGG-SSD); the reference has none of them.  Flatten and Reshape are
// zero-copy views of their bottom with another ncnn rank (Blob::dims).  Parameter ids and defaults follow ncnn.  None of
// them takes part in fusion.
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class PermuteLayer : public Layer {
public:
    explicit PermuteLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        order = pd.get(0, 0);
        if (order < 0 || order > 5) {
            LOGE("Layer %s: Permute order_type %d is not supported (0-5)", this->name.c_str(), order);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    // A rank-2 blob takes order 0 (a view) and 1 (the transpose, how pnnx writes flatten(2).transpose(1, 2)).
    int Reshape() {
        Blob<float>* b = bottoms[0];
        if (b->dims() == 2 && order <= 1) {
            if (order == 0) {
                tops[0]->ViewExternal(b->data(), b->num(), 1, b->height(), b->width(), 2);
            } else {
                tops[0]->ReshapeWithRealloc(b->num(), 1, b->width(), b->height());
                tops[0]->set_dims(2);
            }
            return 0;
        }
        if (b->dims() != 3) {
            LOGE("Layer %s: Permute order_type %d of a rank-%d blob is not supported (rank 3, or rank 2 with order 0 or 1)",
                 this->name.c_str(), order, b->dims());
            return FEATHER_ERR_UNSUPPORTED;
        }
        static const int kAxes[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
        const size_t d[3] = {b->channels(), b->height(), b->width()};
        tops[0]->ReshapeWithRealloc(b->num(), d[kAxes[order][0]], d[kAxes[order][1]], d[kAxes[order][2]]);
        return 0;
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        if (b->dims() == 2 && order == 0) return 0;
        return fcuda_permute_forward(tops[0]->data(), b->data(), static_cast<int>(b->channels()), static_cast<int>(b->height()),
                                     static_cast<int>(b->width()), order, static_cast<int>(b->num()), stream());
    }

private:
    int order = 0;
};

// Rank-1 view of c * h * w floats per image.
class FlattenLayer : public Layer {
public:
    explicit FlattenLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int Reshape() {
        Blob<float>* b = bottoms[0];
        tops[0]->ViewExternal(b->data(), b->num(), 1, 1, b->channels() * b->height() * b->width(), 1);
        return 0;
    }
    int Forward() { return 0; }
};

// ncnn Reshape 0=w 1=h 2=c: the rank is given by which are present (-233 = absent); 0 keeps the bottom's dim of that
// name and -1 infers one dim from the element count.  A view of the bottom.
class ReshapeLayer : public Layer {
public:
    explicit ReshapeLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        w = pd.get(0, -233);
        h = pd.get(1, -233);
        c = pd.get(2, -233);
        if (pd.get(3, 0)) {
            LOGE("Layer %s: Reshape with permute=1 is not supported", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        ndim = w == -233 ? 0 : (h == -233 ? 1 : (c == -233 ? 2 : 3));
        const int v[3] = {w, h, c};
        int inferred = 0;
        for (int i = 0; i < ndim; ++i) {
            if (v[i] < -1) {
                LOGE("Layer %s: Reshape dim %d is not supported", this->name.c_str(), v[i]);
                return FEATHER_ERR_UNSUPPORTED;
            }
            inferred += v[i] == -1;
        }
        if (ndim == 0 || inferred > 1) {
            LOGE("Layer %s: Reshape needs w (0=), and at most one -1", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        Blob<float>* b = bottoms[0];
        const long long total = static_cast<long long>(b->channels()) * b->height() * b->width();
        long long d[3] = {w, h, c};
        const long long keep[3] = {static_cast<long long>(b->width()), static_cast<long long>(b->height()),
                                   static_cast<long long>(b->channels())};
        long long known = 1;
        int infer = -1;
        for (int i = 0; i < ndim; ++i) {
            if (d[i] == 0) d[i] = keep[i];
            if (d[i] == -1) infer = i;
            else known *= d[i];
        }
        if (infer >= 0) d[infer] = known > 0 && total % known == 0 ? total / known : 0;
        long long got = 1;
        for (int i = 0; i < ndim; ++i) got *= d[i];
        if (got != total || got == 0) {
            LOGE("Layer %s: cannot reshape %lld values to w=%lld h=%lld c=%lld", this->name.c_str(), total, d[0],
                 ndim > 1 ? d[1] : 1, ndim > 2 ? d[2] : 1);
            return FEATHER_ERR_TOPOLOGY;
        }
        tops[0]->ViewExternal(b->data(), b->num(), ndim > 2 ? d[2] : 1, ndim > 1 ? d[1] : 1, d[0], ndim);
        return 0;
    }
    int Forward() { return 0; }

private:
    int w = -233, h = -233, c = -233, ndim = 0;
};

class PriorBoxLayer : public Layer {
public:
    explicit PriorBoxLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) { param = FcudaPriorBoxParam(); }
    int LoadParam(const ncnn::ParamDict& pd) {
        // arrays: -23300 min_sizes, -23301 max_sizes, -23302 aspect_ratios (stored at ids 0, 1, 2)
        const ncnn::Mat mins = pd.get(0, ncnn::Mat()), maxs = pd.get(1, ncnn::Mat()), ars = pd.get(2, ncnn::Mat());
        if (mins.w > FCUDA_PRIORBOX_MAX || maxs.w > FCUDA_PRIORBOX_MAX || ars.w > FCUDA_PRIORBOX_MAX) {
            LOGE("Layer %s: PriorBox takes at most %d sizes and aspect ratios", this->name.c_str(), FCUDA_PRIORBOX_MAX);
            return FEATHER_ERR_UNSUPPORTED;
        }
        param.num_min_sizes = mins.empty() ? 0 : mins.w;
        param.num_max_sizes = maxs.empty() ? 0 : maxs.w;
        param.num_aspect_ratios = ars.empty() ? 0 : ars.w;
        for (int i = 0; i < param.num_min_sizes; ++i) param.min_sizes[i] = static_cast<const float*>(mins.data)[i];
        for (int i = 0; i < param.num_max_sizes; ++i) param.max_sizes[i] = static_cast<const float*>(maxs.data)[i];
        for (int i = 0; i < param.num_aspect_ratios; ++i) param.aspect_ratios[i] = static_cast<const float*>(ars.data)[i];
        param.variances[0] = pd.get(3, 0.1f);
        param.variances[1] = pd.get(4, 0.1f);
        param.variances[2] = pd.get(5, 0.2f);
        param.variances[3] = pd.get(6, 0.2f);
        param.flip = pd.get(7, 1);
        param.clip = pd.get(8, 0);
        image_w = pd.get(9, -233);
        image_h = pd.get(10, -233);
        const float sw = pd.get(11, -233.f), sh = pd.get(12, -233.f);
        param.step_w = sw == -233.f ? 0.f : sw;
        param.step_h = sh == -233.f ? 0.f : sh;
        param.offset = pd.get(13, 0.5f);
        if ((sw != -233.f && !(sw > 0.f)) || (sh != -233.f && !(sh > 0.f))) {
            LOGE("Layer %s: PriorBox steps must be positive", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if ((image_w != -233 && image_w < 1) || (image_h != -233 && image_h < 1)) {
            LOGE("Layer %s: PriorBox image size must be positive", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (fcuda_priorbox_per_location(&param, &per_loc) != 0) {
            LOGE("Layer %s: unsupported PriorBox sizes / aspect ratios", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (bottoms.empty() || bottoms.size() > 2 || ((image_w == -233 || image_h == -233) && bottoms.size() != 2)) {
            LOGE("Layer %s: PriorBox takes the feature map and the image as bottoms", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    // The priors depend on shapes only: one image (num 1), read by DetectionOutput for every image of the batch.
    int Reshape() {
        const Blob<float>* feat = bottoms[0];
        fw = static_cast<int>(feat->width());
        fh = static_cast<int>(feat->height());
        iw = image_w != -233 ? image_w : static_cast<int>(bottoms[1]->width());
        ih = image_h != -233 ? image_h : static_cast<int>(bottoms[1]->height());
        const long long priors = static_cast<long long>(fw) * fh * per_loc;
        if (priors < 1 || priors >= (1LL << 24)) {
            LOGE("Layer %s: %lld priors are out of range", this->name.c_str(), priors);
            return FEATHER_ERR_UNSUPPORTED;
        }
        tops[0]->ReshapeWithRealloc(1, 1, 2, static_cast<int>(priors * 4));
        tops[0]->set_dims(2);
        return 0;
    }
    int Forward() { return fcuda_priorbox_forward(tops[0]->data(), &param, fw, fh, iw, ih, stream()); }

    const FcudaPriorBoxParam& prior_param() const { return param; }

private:
    FcudaPriorBoxParam param;
    int per_loc = 0, image_w = -233, image_h = -233;
    int fw = 0, fh = 0, iw = 0, ih = 0;
};

// Bottoms: loc (4 * P per image), conf (P * C per image, class fastest), priors (PriorBox's (2, 4 * P)).  Top: rank 2,
// (keep_top_k, 6) per image, rows [label, score, xmin, ymin, xmax, ymax], padded with label -1 (fcuda.h).
class DetectionOutputLayer : public Layer {
public:
    explicit DetectionOutputLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        num_classes = pd.get(0, 0);
        nms_threshold = pd.get(1, 0.05f);
        nms_top_k = pd.get(2, 300);
        keep_top_k = pd.get(3, 100);
        conf_threshold = pd.get(4, 0.5f);
        if (num_classes < 1 || num_classes > 1024 || nms_top_k < 1 || nms_top_k > 1024 || keep_top_k < 1 ||
            keep_top_k > 1024 || nms_threshold != nms_threshold) {
            LOGE("Layer %s: DetectionOutput needs 1 <= num_classes, nms_top_k, keep_top_k <= 1024", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (bottoms.size() != 3) {
            LOGE("Layer %s: DetectionOutput takes loc, conf and priors", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* loc = bottoms[0];
        const Blob<float>* conf = bottoms[1];
        const Blob<float>* pri = bottoms[2];
        const size_t per_prior = pri->channels() * pri->height() * pri->width();
        if (pri->num() != 1 || pri->channels() != 1 || pri->height() != 2 || pri->width() % 4 != 0) {
            LOGE("Layer %s: the priors blob must be PriorBox's (2, 4 * P)", this->name.c_str());
            return FEATHER_ERR_TOPOLOGY;
        }
        num_priors = static_cast<int>(per_prior / 8);
        const size_t loc_n = loc->channels() * loc->height() * loc->width();
        const size_t conf_n = conf->channels() * conf->height() * conf->width();
        if (loc_n != static_cast<size_t>(num_priors) * 4 || conf_n != static_cast<size_t>(num_priors) * num_classes ||
            loc->num() != conf->num()) {
            LOGE("Layer %s: %zu loc and %zu conf values do not match %d priors of %d classes", this->name.c_str(), loc_n,
                 conf_n, num_priors, num_classes);
            return FEATHER_ERR_TOPOLOGY;
        }
        const int batch = static_cast<int>(loc->num());
        size_t floats = 0;
        const int rc = fcuda_detection_output_workspace_size(num_priors, num_classes, nms_top_k, batch, &floats);
        if (rc) return rc;
        if (!this->common_mempool->Request(sizeof(float) * floats)) return FEATHER_ERR_CUDA;
        tops[0]->ReshapeWithRealloc(batch, 1, keep_top_k, 6);
        tops[0]->set_dims(2);
        return 0;
    }
    int Forward() {
        float* workspace = NULL;
        if (!this->common_mempool->GetPtr(&workspace)) return FEATHER_ERR_CUDA;
        return fcuda_detection_output_forward(tops[0]->data(), bottoms[0]->data(), bottoms[1]->data(), bottoms[2]->data(),
                                              num_priors, num_classes, conf_threshold, nms_threshold, nms_top_k, keep_top_k,
                                              workspace, static_cast<int>(bottoms[0]->num()), stream());
    }

private:
    int num_classes = 0, nms_top_k = 300, keep_top_k = 100, num_priors = 0;
    float nms_threshold = 0.05f, conf_threshold = 0.5f;
};

}  // inline namespace b200
}  // namespace feather
