// YoloDetectionOutputLayer (YOLOv2) and Yolov3DetectionOutputLayer — ncnn's layers of those names, the head of the
// MobileNet-YOLO family; the reference has neither.  Parameter ids and defaults follow ncnn: 0=num_class, 1=num_box,
// 2=confidence_threshold, 3=nms_threshold, -23304=biases, and for v3 -23305=mask, -23306=anchors_scale.  Two ids ncnn does
// not use for these layers cap the work: 20=nms_top_k and 21=keep_top_k (default 1024 each; the output is fixed at
// (keep_top_k, 6) per image, fcuda.h).  Array entries may be written as floats (as ncnn's converters write them) or as
// integers.  Neither layer takes part in fusion.
#pragma once

#include <string.h>

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class YoloDetectionLayerBase : public Layer {
public:
    YoloDetectionLayerBase(RuntimeParameter<float>* rt_param, int version) : Layer(rt_param) {
        memset(&param, 0, sizeof(param));
        param.version = version;
    }
    int LoadParam(const ncnn::ParamDict& pd) {
        const char* type = param.version == 3 ? "Yolov3DetectionOutput" : "YoloDetectionOutput";
        param.num_class = pd.get(0, 20);
        param.num_box = pd.get(1, 5);
        param.confidence_threshold = pd.get(2, 0.01f);
        param.nms_threshold = pd.get(3, 0.45f);
        param.nms_top_k = pd.get(20, 1024);
        param.keep_top_k = pd.get(21, 1024);
        param.num_scales = static_cast<int>(bottoms.size());
        const ncnn::Mat biases = pd.get(4, ncnn::Mat()), mask = pd.get(5, ncnn::Mat()), scales = pd.get(6, ncnn::Mat());
        const int nb = biases.empty() ? 0 : biases.w;
        const int nm = mask.empty() ? 0 : mask.w;
        const int ns = scales.empty() ? 0 : scales.w;
        bool ok = nb <= FCUDA_YOLO_MAX_BIASES && param.num_scales >= 1;
        if (param.version == 3)
            ok = ok && param.num_scales <= FCUDA_YOLO_MAX_SCALES && param.num_box >= 1 &&
                 param.num_box <= FCUDA_YOLO_MAX_BOXES && nm == param.num_box * param.num_scales && ns == param.num_scales;
        if (!ok) {
            LOGE("Layer %s: %s needs <= %d biases, and for v3 1..%d bottoms with num_box mask entries and one anchors_scale "
                 "each", this->name.c_str(), type, FCUDA_YOLO_MAX_BIASES, FCUDA_YOLO_MAX_SCALES);
            return FEATHER_ERR_UNSUPPORTED;
        }
        param.num_biases = nb;
        for (int i = 0; i < nb; ++i) param.biases[i] = value(biases, i);
        for (int i = 0; i < ns && param.version == 3; ++i) param.anchors_scale[i] = value(scales, i);
        for (int i = 0; i < nm && param.version == 3; ++i) {
            const float v = value(mask, i);
            if (!(v >= 0.f && v < 1024.f) || v != static_cast<float>(static_cast<int>(v))) {
                LOGE("Layer %s: mask entry %g is not an anchor index", this->name.c_str(), v);
                return FEATHER_ERR_UNSUPPORTED;
            }
            param.mask[i] = static_cast<int>(v);
        }
        // every limit that does not depend on the bottoms' shapes, on a stand-in 1 x 1 grid
        FcudaYoloParam probe = param;
        for (int b = 0; b < FCUDA_YOLO_MAX_SCALES; ++b) probe.grid_h[b] = probe.grid_w[b] = 1;
        size_t floats = 0;
        if (fcuda_yolo_detection_workspace_size(&probe, 1, &floats) != 0) {
            LOGE("Layer %s: %s parameters out of range (num_class 1..1024, num_box 1..16, %s, nms_top_k / keep_top_k "
                 "1..1024, nms_threshold not NaN)", this->name.c_str(), type,
                 param.version == 3 ? "mask indices within the biases, anchors_scale > 0" : "one bottom, 2 * num_box biases");
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        const size_t want = static_cast<size_t>(param.num_box) * (5 + param.num_class);
        const size_t batch = bottoms[0]->num();
        for (int b = 0; b < param.num_scales; ++b) {
            const Blob<float>* x = bottoms[b];
            if (x->channels() != want || x->num() != batch) {
                LOGE("Layer %s: bottom %d has %zu channels (%zu images), not num_box * (5 + num_class) = %zu (%zu images)",
                     this->name.c_str(), b, x->channels(), x->num(), want, batch);
                return FEATHER_ERR_TOPOLOGY;
            }
            param.grid_h[b] = static_cast<int>(x->height());
            param.grid_w[b] = static_cast<int>(x->width());
        }
        size_t floats = 0;
        const int rc = fcuda_yolo_detection_workspace_size(&param, static_cast<int>(batch), &floats);
        if (rc) {
            LOGE("Layer %s: %zu images of these grids are out of range", this->name.c_str(), batch);
            return rc;
        }
        if (!this->common_mempool->Request(sizeof(float) * floats)) return FEATHER_ERR_CUDA;
        tops[0]->ReshapeWithRealloc(batch, 1, param.keep_top_k, 6);
        tops[0]->set_dims(2);
        return 0;
    }
    int Forward() {
        float* workspace = NULL;
        if (!this->common_mempool->GetPtr(&workspace)) return FEATHER_ERR_CUDA;
        const float* inputs[FCUDA_YOLO_MAX_SCALES] = {};
        for (int b = 0; b < param.num_scales; ++b) inputs[b] = bottoms[b]->data();
        return fcuda_yolo_detection_forward(tops[0]->data(), inputs, &param, workspace, static_cast<int>(bottoms[0]->num()),
                                            stream());
    }

private:
    // An array entry written as an integer holds the int's bits: a nonzero value below 2^23 reads as a denormal float.
    static float value(const ncnn::Mat& m, int i) {
        const float f = static_cast<const float*>(m.data)[i];
        const int bits = static_cast<const int*>(m.data)[i];
        return bits > 0 && bits < (1 << 23) ? static_cast<float>(bits) : f;
    }

    FcudaYoloParam param;
};

class YoloDetectionOutputLayer : public YoloDetectionLayerBase {
public:
    explicit YoloDetectionOutputLayer(RuntimeParameter<float>* rt_param) : YoloDetectionLayerBase(rt_param, 2) {}
};

class Yolov3DetectionOutputLayer : public YoloDetectionLayerBase {
public:
    explicit Yolov3DetectionOutputLayer(RuntimeParameter<float>* rt_param) : YoloDetectionLayerBase(rt_param, 3) {}
};

}  // inline namespace b200
}  // namespace feather
