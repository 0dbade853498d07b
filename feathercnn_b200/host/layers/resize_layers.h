// InterpLayer and CropLayer — serve ncnn "Interp" (nearest / bilinear resize) and "Crop", the layers segmentation heads
// use to bring logits back to the input size (the reference has neither).  Net::ApplyFusion folds a Crop of a
// deconvolution's otherwise unread output into the deconvolution's pads (DeconvLayer::FoldCrop).
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class InterpLayer : public Layer {
public:
    explicit InterpLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) { param = FcudaInterpParam(); }

    int LoadParam(const ncnn::ParamDict& pd) {
        // ncnn's Interp parameter ids
        param.resize_type = pd.get(0, 0);
        param.height_scale = pd.get(1, 1.f);
        param.width_scale = pd.get(2, 1.f);
        param.output_height = pd.get(3, 0);
        param.output_width = pd.get(4, 0);
        param.align_corner = pd.get(6, 0);
        if (pd.get(5, 0)) {
            LOGE("Layer %s: dynamic_target_size (the size of a second blob) is not supported", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (bottoms.size() != 1) {
            LOGE("Layer %s: Interp takes one bottom blob", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (param.resize_type != 1 && param.resize_type != 2) {
            LOGE("Layer %s: resize_type %d is not supported (1 nearest, 2 bilinear)", this->name.c_str(), param.resize_type);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }

    int Reshape() {
        const Blob<float>* bottom = bottoms[0];
        param.input_h = static_cast<int>(bottom->height());
        param.input_w = static_cast<int>(bottom->width());
        const int rc = fcuda_interp_output_dim(&param);
        if (rc) return rc;
        tops[0]->ReshapeWithRealloc(bottom->num(), bottom->channels(), param.output_h, param.output_w);
        return 0;
    }

    int Forward() {
        const Blob<float>* bottom = bottoms[0];
        return fcuda_interp_forward(&param, tops[0]->data(), bottom->data(), static_cast<int>(bottom->channels()),
                                    static_cast<int>(bottom->num()), stream());
    }

    // ncnn's parameters; input_h / input_w and the output size are those of the last Reshape
    const FcudaInterpParam& interp_param() const { return param; }

private:
    FcudaInterpParam param;
};

// The window of a Crop in (c, h, w): offsets and sizes.  A second bottom, when present, gives the output height and
// width and is never read; channels are cropped by coffset / outc only (Caffe's Crop with axis 2).
struct CropWindow {
    int coff = 0, hoff = 0, woff = 0;
    int outc = 0, outh = 0, outw = 0;  // 0: to the end of that axis (one bottom)

    // resolves the sizes against the input (and reference) shape; false when the window does not fit
    bool Resolve(int c, int h, int w, const Blob<float>* reference, int* oc, int* oh, int* ow) const {
        *oc = outc ? outc : c - coff;
        *oh = reference ? static_cast<int>(reference->height()) : (outh ? outh : h - hoff);
        *ow = reference ? static_cast<int>(reference->width()) : (outw ? outw : w - woff);
        return *oc > 0 && *oh > 0 && *ow > 0 && coff + *oc <= c && hoff + *oh <= h && woff + *ow <= w;
    }
};

class CropLayer : public Layer {
public:
    explicit CropLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}

    int LoadParam(const ncnn::ParamDict& pd) {
        // ncnn's Crop parameter ids
        win.woff = pd.get(0, 0);
        win.hoff = pd.get(1, 0);
        win.coff = pd.get(2, 0);
        win.outw = pd.get(3, 0);
        win.outh = pd.get(4, 0);
        win.outc = pd.get(5, 0);
        // end offsets (6-8) and the slice form (9 starts, 10 ends, 11 axes) would select another window
        for (int id = 6; id <= 8; ++id)
            if (pd.get(id, 0)) {
                LOGE("Layer %s: Crop parameter %d (end offsets) is not supported", this->name.c_str(), id);
                return FEATHER_ERR_UNSUPPORTED;
            }
        for (int id = 9; id <= 11; ++id)
            if (!pd.get(id, ncnn::Mat()).empty()) {
                LOGE("Layer %s: Crop parameter %d (starts / ends / axes) is not supported", this->name.c_str(), id);
                return FEATHER_ERR_UNSUPPORTED;
            }
        if (win.woff < 0 || win.hoff < 0 || win.coff < 0 || win.outw < 0 || win.outh < 0 || win.outc < 0) {
            LOGE("Layer %s: negative Crop offsets or sizes are not supported", this->name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (bottoms.empty() || bottoms.size() > 2) return FEATHER_ERR_UNSUPPORTED;
        return 0;
    }

    int Reshape() {
        const Blob<float>* bottom = bottoms[0];
        if (!win.Resolve(static_cast<int>(bottom->channels()), static_cast<int>(bottom->height()),
                         static_cast<int>(bottom->width()), reference(), &oc, &oh, &ow)) {
            LOGE("Layer %s: the crop window does not fit its %zux%zux%zu input", this->name.c_str(), bottom->channels(),
                 bottom->height(), bottom->width());
            return FEATHER_ERR_TOPOLOGY;
        }
        tops[0]->ReshapeWithRealloc(bottom->num(), oc, oh, ow);
        return 0;
    }

    int Forward() {
        const Blob<float>* b = bottoms[0];
        return fcuda_crop_forward(tops[0]->data(), b->data(), static_cast<int>(b->channels()), static_cast<int>(b->height()),
                                  static_cast<int>(b->width()), win.coff, win.hoff, win.woff, oc, oh, ow,
                                  static_cast<int>(b->num()), stream());
    }

    const CropWindow& window() const { return win; }
    Blob<float>* reference() const { return bottoms.size() > 1 ? bottoms[1] : NULL; }

private:
    CropWindow win;
    int oc = 0, oh = 0, ow = 0;
};

}  // inline namespace b200
}  // namespace feather
