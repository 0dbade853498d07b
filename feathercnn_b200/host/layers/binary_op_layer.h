// BinaryOpLayer: ncnn's BinaryOp (the reference has no such layer), which onnx2ncnn writes for ONNX Add / Sub / Mul /
// Div / Max / Min / Pow and pnnx for torch.add, x + y, x * 0.5 and the like.  Element-wise op of two bottoms, or of one
// bottom and the scalar 2=, with the operand rule of fcuda_binary_op_shape.  A following ReLU joins it (Fuse), and
// Net::ApplyFusion treats an ADD of two bottoms like a plain Eltwise SUM (a residual or super-resolution tail add).
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// 0 = op_type (0 ADD .. 11 RATAN2, FcudaBinaryOp), 1 = with_scalar (0: two bottoms; 1: one bottom and 2=), 2 = b (0.0).
// No weights.
class BinaryOpLayer : public Layer {
public:
    explicit BinaryOpLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) { _fusible = true; }
    int LoadParam(const ncnn::ParamDict& pd) {
        op_type = pd.get(0, 0);
        with_scalar = pd.get(1, 0);
        b = pd.get(2, 0.f);
        if (op_type < FCUDA_BINARY_ADD || op_type > FCUDA_BINARY_RATAN2 || (with_scalar != 0 && with_scalar != 1) ||
            bottoms.size() != (with_scalar ? 1u : 2u) || tops.size() != 1) {
            LOGE("BinaryOp layer %s: op_type %d, with_scalar %d with %zu bottoms and %zu tops is not supported (op_type "
                 "0..11; one bottom with with_scalar=1, two otherwise; one top)", this->name.c_str(), op_type,
                 with_scalar, bottoms.size(), tops.size());
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* x = bottoms[0];
        if (with_scalar) {
            tops[0]->ReshapeWithRealloc(x);
            return 0;
        }
        const Blob<float>* y = bottoms[1];
        const int xs[3] = {static_cast<int>(x->channels()), static_cast<int>(x->height()), static_cast<int>(x->width())};
        const int ys[3] = {static_cast<int>(y->channels()), static_cast<int>(y->height()), static_cast<int>(y->width())};
        int rank = 0, out[3];
        if (x->num() != y->num() ||
            fcuda_binary_op_shape(x->dims(), xs, y->dims(), ys, &rank, out, a_shape + 1, b_shape + 1) != 0) {
            LOGE("BinaryOp layer %s: %s (%zu, %zu, %zu, %zu) rank %d and %s (%zu, %zu, %zu, %zu) rank %d do not broadcast",
                 this->name.c_str(), x->name.c_str(), x->num(), x->channels(), x->height(), x->width(), x->dims(),
                 y->name.c_str(), y->num(), y->channels(), y->height(), y->width(), y->dims());
            return FEATHER_ERR_TOPOLOGY;
        }
        a_shape[0] = b_shape[0] = static_cast<int>(x->num());
        tops[0]->ReshapeWithRealloc(a_shape[0], out[0], out[1], out[2]);
        tops[0]->set_dims(rank);
        return 0;
    }
    int Forward() {
        const Blob<float>* x = bottoms[0];
        if (with_scalar) {
            const int s[4] = {static_cast<int>(x->num()), static_cast<int>(x->channels()), static_cast<int>(x->height()),
                              static_cast<int>(x->width())};
            return fcuda_binary_op_forward(tops[0]->data(), x->data(), s, NULL, NULL, b, op_type, relu, stream());
        }
        return fcuda_binary_op_forward(tops[0]->data(), x->data(), a_shape, bottoms[1]->data(), b_shape, 0.f, op_type,
                                       relu, stream());
    }
    int Fuse(Layer* next_layer) {
        if (next_layer->type.compare("ReLU") == 0 && !relu) {
            relu = 1;
            return 1;
        }
        return 0;
    }

    // An ADD of two bottoms: what Net::ApplyFusion's residual and tail passes take like a plain Eltwise SUM.
    bool plain_add() const { return op_type == FCUDA_BINARY_ADD && !with_scalar; }
    int fused_relu() const { return relu; }

private:
    int op_type = 0, with_scalar = 0, relu = 0;
    float b = 0.f;
    int a_shape[4] = {0, 0, 0, 0}, b_shape[4] = {0, 0, 0, 0};  // (n, c, h, w) along the output's axes (Reshape)
};

}  // inline namespace b200
}  // namespace feather
