// PixelShuffleLayer: ncnn's PixelShuffle, the sub-pixel upsampling that ends super-resolution nets (Real-ESRGAN's
// SRVGGNetCompact, EDSR; the reference has no such layer).  Net::ApplyFusion may hand it SRVGGNetCompact's tail: an
// Eltwise SUM of its output and a nearest Interp of another blob, which it then adds in the same pass
// (fcuda_pixel_shuffle_forward with an addend), so neither the Interp's output nor its own is written.
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// 0 = upscale_factor (1), 1 = mode (0: PyTorch's channel order, 1: ONNX DepthToSpace DCR).  No weights.
class PixelShuffleLayer : public Layer {
public:
    explicit PixelShuffleLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        r = pd.get(0, 1);
        mode = pd.get(1, 0);
        if (r < 1 || (mode != 0 && mode != 1)) {
            LOGE("PixelShuffle layer %s: upscale_factor %d, mode %d is not supported", this->name.c_str(), r, mode);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* b = bottoms[0];
        const size_t rr = static_cast<size_t>(r) * r;
        if (b->channels() % rr) {
            LOGE("PixelShuffle layer %s: %zu channels is not a multiple of %zu", this->name.c_str(), b->channels(), rr);
            return FEATHER_ERR_TOPOLOGY;
        }
        const size_t oc = b->channels() / rr, oh = b->height() * r, ow = b->width() * r;
        if (base) {  // the fused tail: the Interp's map of the addend must land on this output
            tail_map.input_h = static_cast<int>(base->height());
            tail_map.input_w = static_cast<int>(base->width());
            if (fcuda_interp_output_dim(&tail_map) || base->num() != b->num() || base->channels() != oc ||
                static_cast<size_t>(tail_map.output_h) != oh || static_cast<size_t>(tail_map.output_w) != ow) {
                LOGE("PixelShuffle layer %s: the added blob %s does not upsample to %zu x %zu x %zu", this->name.c_str(),
                     base->name.c_str(), oc, oh, ow);
                return FEATHER_ERR_TOPOLOGY;
            }
        }
        tops[0]->ReshapeWithRealloc(b->num(), oc, oh, ow);
        return 0;
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        return fcuda_pixel_shuffle_forward(tops[0]->data(), b->data(), static_cast<int>(b->channels()),
                                           static_cast<int>(b->height()), static_cast<int>(b->width()), r, mode,
                                           base ? base->data() : NULL, base ? &tail_map : NULL,
                                           static_cast<int>(b->num()), stream());
    }
    // Adds the nearest Interp `map` of `addend` to the output (SRVGGNetCompact's tail); `addend` must be computed before
    // this layer runs.  Returns 1 when taken: a nearest map, and no tail taken before.
    int FuseUpsampledAdd(const FcudaInterpParam& map, Blob<float>* addend) {
        if (base || map.resize_type != 1 || !addend) return 0;
        tail_map = map;
        base = addend;
        return 1;
    }

private:
    int r = 1, mode = 0;
    Blob<float>* base = NULL;  // the fused tail's addend, before its Interp
    FcudaInterpParam tail_map = FcudaInterpParam();
};

}  // inline namespace b200
}  // namespace feather
