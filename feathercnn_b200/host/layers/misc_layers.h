// Input, Split, Concat, Softmax, Dropout layers (mirror /root/reference/src/layers/input_layer.h:25-52,
// split_layer.h:22-54, concat_layer.h:22-83, softmax_layer.h:24-57, dropout_layer.h:22-60).
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class InputLayer : public Layer {
public:
    explicit InputLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param), w(0), h(0), c(0) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        w = pd.get(0, 0);
        h = pd.get(1, 0);
        c = pd.get(2, 0);
        return 0;
    }
    int Reshape() { return 0; }  // shape comes from FeedInput (input_layer.h:40-44)
    int Init() { return 0; }
    int w, h, c;  // declared input shape, used by the README-era Forward(float*)
};

// Split: the reference memcpy()s the bottom into every top (split_layer.h:43-53).  No layer in this engine
// writes into its bottoms, so the tops are zero-copy views of the bottom instead.
class SplitLayer : public Layer {
public:
    explicit SplitLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int Reshape() {
        const Blob<float>* b = bottoms[0];
        for (size_t i = 0; i < tops.size(); ++i) tops[i]->ViewExternal(b->data(), b->num(), b->channels(), b->height(), b->width(), b->dims());
        return 0;
    }
    int Forward() { return 0; }
};

class ConcatLayer : public Layer {
public:
    explicit ConcatLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param), axis(0) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        this->axis = pd.get(0, 0);
        return 0;
    }
    // ncnn axis of a 3-D blob: 0 = channels, 1 = height, 2 = width.  The reference handles axis 0 only
    // (concat_layer.h:50-54); 1 and 2 are this engine's extension (SURVEY.md §8f rank 4).  Rank-1 and rank-2 bottoms
    // (SSD's flattened heads and prior boxes) take ncnn's per-rank axis: rank 1: 0 = w; rank 2: 0 = h, 1 = w; a negative
    // axis adds the rank.
    int Reshape() {
        const Blob<float>* first_blob = this->bottoms[0];
        const int rank = first_blob->dims();
        int a = axis;
        if (rank != 3 && a < 0) a += rank;
        if (a < 0 || a >= rank) {
            LOGE("Concat layer %s: unsupported axis %d for rank %d", this->name.c_str(), axis, rank);
            return FEATHER_ERR_WEIGHTS;
        }
        storage_axis = a + 3 - rank;
        size_t dims[3] = {first_blob->channels(), first_blob->height(), first_blob->width()};
        const size_t num = first_blob->num();
        for (size_t i = 1; i < bottoms.size(); ++i) {
            const Blob<float>* p_blob = bottoms[i];
            const size_t d[3] = {p_blob->channels(), p_blob->height(), p_blob->width()};
            if (p_blob->dims() != rank) {
                LOGE("Concat layer %s: bottoms of ranks %d and %d", this->name.c_str(), rank, p_blob->dims());
                return FEATHER_ERR_WEIGHTS;
            }
            for (int k = 0; k < 3; ++k)
                if (k != storage_axis && d[k] != dims[k]) {
                    LOGE("Images of different shapes cannot be concatenated together");
                    return FEATHER_ERR_WEIGHTS;
                }
            if (num != p_blob->num()) return FEATHER_ERR_WEIGHTS;
            dims[storage_axis] += d[storage_axis];
        }
        tops[0]->ReshapeWithRealloc(num, dims[0], dims[1], dims[2]);
        tops[0]->set_dims(rank);
        return 0;
    }
    int Forward() {
        // [outer][mid][inner] copy: outer = everything before the axis, mid = the axis, inner = everything after it
        int offset = 0, rc = 0;
        const Blob<float>* t = tops[0];
        for (size_t i = 0; i < bottoms.size() && rc == 0; ++i) {
            const Blob<float>* b = bottoms[i];
            size_t outer, mid, dst_mid, inner;
            if (storage_axis == 0) { outer = b->num(); mid = b->channels(); dst_mid = t->channels(); inner = t->height() * t->width(); }
            else if (storage_axis == 1) { outer = b->num() * b->channels(); mid = b->height(); dst_mid = t->height(); inner = t->width(); }
            else { outer = b->num() * b->channels() * b->height(); mid = b->width(); dst_mid = t->width(); inner = 1; }
            rc = fcuda_copy_channels(t->data(), static_cast<int>(dst_mid), offset, b->data(), static_cast<int>(mid), inner,
                                     static_cast<int>(outer), stream());
            offset += static_cast<int>(mid);
        }
        return rc;
    }
    int param_axis() const { return axis; }

private:
    int axis;
    int storage_axis = 0;  // axis of the (c, h, w) storage
};

// Without 0= on its line: the reference's softmax over each image's whole blob.  With 0=axis: ncnn's softmax over that
// axis of the blob's rank (rank 1: 0 = w; rank 2: 0 = h, 1 = w; rank 3: 0 = c, 1 = h, 2 = w; negative adds the rank).
// 1= (ncnn's fixbug0) is accepted and ignored.
class SoftmaxLayer : public Layer {
public:
    explicit SoftmaxLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        has_axis = pd.has(0);
        axis = pd.get(0, 0);
        return 0;
    }
    int Reshape() {
        if (has_axis) {
            const int rank = bottoms[0]->dims();
            const int a = axis < 0 ? axis + rank : axis;
            if (a < 0 || a >= rank) {
                LOGE("Softmax layer %s: axis %d is out of range for rank %d", this->name.c_str(), axis, rank);
                return FEATHER_ERR_UNSUPPORTED;
            }
            storage_axis = a + 3 - rank;
        }
        return Layer::Reshape();
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        if (!has_axis)
            return fcuda_softmax_forward(tops[0]->data(), b->data(), b->channels() * b->height() * b->width(), b->num(), stream());
        const size_t d[3] = {b->channels(), b->height(), b->width()};
        size_t outer = 1, inner = 1;
        for (int k = 0; k < storage_axis; ++k) outer *= d[k];
        for (int k = storage_axis + 1; k < 3; ++k) inner *= d[k];
        return fcuda_softmax_axis_forward(tops[0]->data(), b->data(), static_cast<int>(outer), static_cast<int>(d[storage_axis]),
                                          static_cast<int>(inner), static_cast<int>(b->num()), stream());
    }
    bool whole_blob() const { return !has_axis; }

private:
    bool has_axis = false;
    int axis = 0;
    int storage_axis = 0;
};

class DropoutLayer : public Layer {
public:
    explicit DropoutLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param), scale(1.f) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        scale = pd.get(0, 1.f);
        return 0;
    }
    int Reshape() {
        const Blob<float>* b = bottoms[0];
        if (scale == 1.f) {  // the reference memcpy()s (dropout_layer.h:40-43); a view is equivalent
            tops[0]->ViewExternal(b->data(), b->num(), b->channels(), b->height(), b->width(), b->dims());
            return 0;
        }
        tops[0]->ReshapeWithRealloc(b);
        return 0;
    }
    int Forward() {
        if (scale == 1.f) return 0;
        return fcuda_dropout_forward(tops[0]->data(), bottoms[0]->data(), bottoms[0]->data_size(), scale, stream());
    }

private:
    float scale;
};

}  // inline namespace b200
}  // namespace feather
