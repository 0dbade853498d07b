// feather::Layer base class (mirrors /root/reference/src/layer.cpp:22-142).
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

Layer::Layer(RuntimeParameter<float>* rt_param)
    : _fusible(false), _inplace(false), common_mempool(rt_param->common_mempool()), rt_param(rt_param) {}

Layer::~Layer() {
    if (!_inplace)
        for (size_t i = 0; i < tops.size(); ++i) delete tops[i];
    for (size_t i = 0; i < weights.size(); ++i) delete weights[i];
}

int Layer::FindBottomIDByName(std::string name) {
    for (size_t i = 0; i < bottoms.size(); ++i)
        if (bottoms[i]->name.compare(name) == 0) return static_cast<int>(i);
    return -1;
}

int Layer::FindTopIDByName(std::string name) {
    for (size_t i = 0; i < tops.size(); ++i)
        if (tops[i]->name.compare(name) == 0) return static_cast<int>(i);
    return -1;
}

int Layer::LoadParam(const ncnn::ParamDict&) { return 0; }
int Layer::LoadWeights(const ncnn::ModelBin&) { return 0; }

int Layer::TryFuse(Layer* next_layer) {
    // fuse only when next_layer consumes one of this layer's tops (layer.cpp:82-96)
    for (size_t i = 0; i < next_layer->bottoms.size(); ++i)
        for (size_t j = 0; j < tops.size(); ++j)
            if (tops[j]->name.compare(next_layer->bottoms[i]->name) == 0) return Fuse(next_layer);
    return 0;
}

int Layer::Fuse(Layer*) { return 0; }

int Layer::Reshape() {
    // default: one top shaped like the single bottom (layer.cpp:103-114)
    if (tops.size() != 1 || bottoms.size() != 1) return FEATHER_ERR_BASE_LAYER;
    tops[0]->ReshapeWithRealloc(bottoms[0]);
    return 0;
}

int Layer::Init() { return 0; }
int Layer::Forward() { return 0; }

int Layer::ForwardReshape() {
    tops[0]->ReshapeWithRealloc(bottoms[0]);
    return this->Forward();
}

bool Layer::fusible() const { return _fusible; }

Blob<float>* Layer::NewWeightBlob(const std::string& blob_name, int n, int c, int h, int w) {
    Blob<float>* b = new Blob<float>(blob_name);
    b->StageOnHost(true);
    b->ReshapeWithRealloc(n, c, h, w);
    return b;
}

}  // inline namespace b200
}  // namespace feather
