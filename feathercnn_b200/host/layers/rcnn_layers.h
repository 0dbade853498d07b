// ProposalLayer, ROIPoolingLayer and PSROIPoolingLayer — ncnn's Proposal, ROIPooling and PSROIPooling, the layers of a
// Faster R-CNN and an R-FCN the other layers do not cover; the reference has none of them.  Parameter ids and defaults
// follow ncnn: Proposal 0=feat_stride (16) 1=base_size (16) 2=pre_nms_topN (6000) 3=after_nms_topN (300) 4=nms_thresh
// (0.7) 5=min_size (16); ROIPooling 0=pooled_w (7) 1=pooled_h (7) 2=spatial_scale (0.0625); PSROIPooling the same and
// 3=output_dim (0, which is rejected: a net must give it).  Proposal's output has a fixed shape (include/fcuda.h): rois
// (after_nms_topN, 1, 4) per image, zero rows past the kept count, and an optional second top of scores (after_nms_topN,
// 1, 1), -1 past the count.  ROIPooling and PSROIPooling pool every RoI of image n from image n's map, so their tops have
// batch * after_nms_topN items and the layers after them (fc6, fc7, ...; R-FCN's average-pooling vote) run once over all
// of them.  None of these layers takes part in fusion.
#pragma once

#include <math.h>

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class ProposalLayer : public Layer {
public:
    explicit ProposalLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        param.feat_stride = pd.get(0, 16);
        param.base_size = pd.get(1, 16);
        param.pre_nms_topN = pd.get(2, 6000);
        param.after_nms_topN = pd.get(3, 300);
        param.nms_thresh = pd.get(4, 0.7f);
        param.min_size = pd.get(5, 16);
        size_t floats = 0;
        if (bottoms.size() != 3 || tops.empty() || tops.size() > 2 ||
            fcuda_proposal_workspace_size(&param, 1, 1, 1, &floats) != 0) {
            LOGE("Layer %s: Proposal needs 3 bottoms (score, bbox, im_info), 1 or 2 tops, feat_stride and base_size >= 1, "
                 "pre_nms_topN and after_nms_topN in 1..8192 and nms_thresh not NaN", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* score = bottoms[0];
        const Blob<float>* bbox = bottoms[1];
        const Blob<float>* info = bottoms[2];
        const size_t A = FCUDA_PROPOSAL_ANCHORS, batch = score->num();
        if (score->channels() != 2 * A || bbox->channels() != 4 * A || bbox->height() != score->height() ||
            bbox->width() != score->width() || bbox->num() != batch || info->num() != batch ||
            info->channels() * info->height() * info->width() != 3) {
            LOGE("Layer %s: Proposal needs score (%zu, H, W), bbox (%zu, H, W) and im_info (3 values) per image, all of "
                 "one batch", this->name.c_str(), 2 * A, 4 * A);
            return FEATHER_ERR_TOPOLOGY;
        }
        feat_h = static_cast<int>(score->height());
        feat_w = static_cast<int>(score->width());
        size_t floats = 0;
        const int rc = fcuda_proposal_workspace_size(&param, feat_h, feat_w, static_cast<int>(batch), &floats);
        if (rc) {
            LOGE("Layer %s: %zu images of a %d x %d map are out of range", this->name.c_str(), batch, feat_h, feat_w);
            return rc;
        }
        if (!this->common_mempool->Request(sizeof(float) * floats)) return FEATHER_ERR_CUDA;
        tops[0]->ReshapeWithRealloc(batch, param.after_nms_topN, 1, 4);
        if (tops.size() > 1) tops[1]->ReshapeWithRealloc(batch, param.after_nms_topN, 1, 1);
        return 0;
    }
    int Forward() {
        float* workspace = NULL;
        if (!this->common_mempool->GetPtr(&workspace)) return FEATHER_ERR_CUDA;
        return fcuda_proposal_forward(tops[0]->data(), tops.size() > 1 ? tops[1]->data() : NULL, bottoms[0]->data(),
                                      bottoms[1]->data(), bottoms[2]->data(), &param, feat_h, feat_w, workspace,
                                      static_cast<int>(bottoms[0]->num()), stream());
    }

private:
    FcudaProposalParam param = {};
    int feat_h = 0, feat_w = 0;
};

class ROIPoolingLayer : public Layer {
public:
    explicit ROIPoolingLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        pooled_w = pd.get(0, 7);
        pooled_h = pd.get(1, 7);
        spatial_scale = pd.get(2, 0.0625f);
        if (bottoms.size() != 2 || pooled_w < 1 || pooled_h < 1 || !isfinite(spatial_scale) || !(spatial_scale > 0.f)) {
            LOGE("Layer %s: ROIPooling needs 2 bottoms (feature map, rois), pooled_w and pooled_h >= 1 and a finite "
                 "spatial_scale > 0", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* x = bottoms[0];
        const Blob<float>* rois = bottoms[1];
        if (rois->num() != x->num() || rois->height() * rois->width() != 4) {
            LOGE("Layer %s: ROIPooling needs rois (R, 1, 4) per image of the feature map's batch", this->name.c_str());
            return FEATHER_ERR_TOPOLOGY;
        }
        tops[0]->ReshapeWithRealloc(x->num() * rois->channels(), x->channels(), pooled_h, pooled_w);
        return 0;
    }
    int Forward() {
        const Blob<float>* x = bottoms[0];
        return fcuda_roi_pooling_forward(tops[0]->data(), x->data(), bottoms[1]->data(), static_cast<int>(x->channels()),
                                         static_cast<int>(x->height()), static_cast<int>(x->width()),
                                         static_cast<int>(bottoms[1]->channels()), pooled_h, pooled_w, spatial_scale,
                                         static_cast<int>(x->num()), stream());
    }

private:
    int pooled_w = 7, pooled_h = 7;
    float spatial_scale = 0.0625f;
};

class PSROIPoolingLayer : public Layer {
public:
    explicit PSROIPoolingLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        pooled_w = pd.get(0, 7);
        pooled_h = pd.get(1, 7);
        spatial_scale = pd.get(2, 0.0625f);
        output_dim = pd.get(3, 0);
        if (bottoms.size() != 2 || pooled_w < 1 || pooled_h < 1 || output_dim < 1 || !isfinite(spatial_scale) ||
            !(spatial_scale > 0.f)) {
            LOGE("Layer %s: PSROIPooling needs 2 bottoms (score maps, rois), pooled_w, pooled_h and output_dim >= 1 and "
                 "a finite spatial_scale > 0", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* x = bottoms[0];
        const Blob<float>* rois = bottoms[1];
        if (x->channels() != static_cast<size_t>(output_dim) * pooled_h * pooled_w) {
            LOGE("Layer %s: PSROIPooling needs output_dim x pooled_h x pooled_w = %d x %d x %d channels, not %zu",
                 this->name.c_str(), output_dim, pooled_h, pooled_w, x->channels());
            return FEATHER_ERR_TOPOLOGY;
        }
        if (rois->num() != x->num() || rois->height() * rois->width() != 4) {
            LOGE("Layer %s: PSROIPooling needs rois (R, 1, 4) per image of the score maps' batch", this->name.c_str());
            return FEATHER_ERR_TOPOLOGY;
        }
        tops[0]->ReshapeWithRealloc(x->num() * rois->channels(), output_dim, pooled_h, pooled_w);
        return 0;
    }
    int Forward() {
        const Blob<float>* x = bottoms[0];
        return fcuda_psroi_pooling_forward(tops[0]->data(), x->data(), bottoms[1]->data(), static_cast<int>(x->channels()),
                                           static_cast<int>(x->height()), static_cast<int>(x->width()),
                                           static_cast<int>(bottoms[1]->channels()), pooled_h, pooled_w, output_dim,
                                           spatial_scale, static_cast<int>(x->num()), stream());
    }

private:
    int pooled_w = 7, pooled_h = 7, output_dim = 0;
    float spatial_scale = 0.0625f;
};

}  // inline namespace b200
}  // namespace feather
