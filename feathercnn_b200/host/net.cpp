// feather::Net (see include/feather/net.h).  Load / Forward structure follows the reference
// (/root/reference/src/net.cpp:31-350): LoadParam builds the layer graph by blob name, LoadWeights streams the
// .bin into the layers in file order, Forward = Reshape-all -> lazy Init-all -> Forward-all.
#include <feather/net.h>

#include <cuda_runtime.h>
#include <fcuda.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <feather/layer_factory.h>

#include "layers/conv_layer.h"
#include "layers/binary_op_layer.h"
#include "layers/deconv_layer.h"
#include "layers/eltwise_layer.h"
#include "layers/misc_layers.h"
#include "layers/pixel_shuffle_layer.h"
#include "layers/resize_layers.h"
#include "layers/route_layers.h"
#include "layers/transformer_layers.h"

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

static const char kContainerMagic[8] = {'F', 'T', 'H', 'R', 'B', '2', '0', '0'};
static const int kMaxLayers = 1 << 20;  // sanity bound on counts read from a .param (a corrupt file must not drive resize())

#define CUDA_OK(expr)                                                                        \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            LOGE("%s failed: %s", #expr, cudaGetErrorString(_e));                            \
            return FEATHER_ERR_CUDA;                                                         \
        }                                                                                    \
    } while (0)

Net::Net() : _param_loaded(0), _weights_loaded(0), _net_initialized(0) {
    register_layer_creators();
    CommonMemPool<float>* mempool = new CommonMemPool<float>();
    rt_param = new RuntimeParameter<float>(mempool, 1);
    int dev = 0;
    cudaGetDevice(&dev);
    rt_param->set_device(dev);
    cudaStream_t s = nullptr;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess) {
        rt_param->set_stream(s);
        owns_stream_ = true;
    }
}

Net::Net(size_t) : Net() {}

Net::~Net() {
    ResetGraph();
    FreePipeline();
    for (size_t i = 0; i < layers.size(); ++i) {
        delete layers[i];
        layers[i] = NULL;
    }
    if (weight_arena_) cudaFree(weight_arena_);
    if (pixel_stage_) cudaFree(pixel_stage_);
    if (owns_stream_ && rt_param->stream()) cudaStreamDestroy(static_cast<cudaStream_t>(rt_param->stream()));
    delete rt_param->common_mempool();
    delete rt_param;
    rt_param = NULL;
}

void Net::SetStream(void* cuda_stream) {
    ResetGraph();
    if (owns_stream_ && rt_param->stream()) cudaStreamDestroy(static_cast<cudaStream_t>(rt_param->stream()));
    owns_stream_ = false;
    rt_param->set_stream(cuda_stream);
}

// ---------------------------------------------------------------------------------------------------------
// Loading
// ---------------------------------------------------------------------------------------------------------
int Net::LoadParam(const char* path) {
    FILE* fp = fopen(path, "r");
    if (fp == NULL) {
        LOGE("Cannot open param file, path: %s", path);
        return -1;
    }
    const int rc = this->LoadParam(fp);
    fclose(fp);
    return rc;
}

int Net::LoadParam(FILE* param_fp) {
    fseek(param_fp, 0, SEEK_END);
    const long len = ftell(param_fp);
    fseek(param_fp, 0, SEEK_SET);
    if (len <= 0) return -1;
    std::string text(static_cast<size_t>(len), '\0');
    if (fread(&text[0], 1, text.size(), param_fp) != text.size()) return -1;
    return ParseParamText(text.c_str());
}

int Net::LoadParamFromText(const char* param_text) { return param_text ? ParseParamText(param_text) : -1; }

int Net::ParseParamText(const char* mem) {
    int consumed = 0, magic = 0;
    if (sscanf(mem, "%d%n", &magic, &consumed) != 1) {
        LOGE("issue with param file");
        return -1;
    }
    mem += consumed;
    if (magic != 7767517) {  // utils.cpp:27-43
        LOGE("param is too old, please regenerate");
        return -1;
    }
    int layer_count = 0, blob_count = 0;
    if (sscanf(mem, "%d %d%n", &layer_count, &blob_count, &consumed) != 2 || layer_count <= 0 || blob_count <= 0 ||
        layer_count > kMaxLayers || blob_count > kMaxLayers) {
        LOGE("issue with param file");
        return -1;
    }
    mem += consumed;
    layers.assign(static_cast<size_t>(layer_count), NULL);
    ncnn::ParamDict pd;
    for (int i = 0; i < layer_count; i++) {
        char layer_type[257], layer_name[257];
        int bottom_count = 0, top_count = 0;
        if (sscanf(mem, "%256s %256s %d %d%n", layer_type, layer_name, &bottom_count, &top_count, &consumed) != 4) {
            LOGE("param file ends after %d of %d layers", i, layer_count);
            return -1;
        }
        if (bottom_count < 0 || top_count < 0 || bottom_count > kMaxLayers || top_count > kMaxLayers) {
            LOGE("layer %s: bad bottom/top count (%d, %d)", layer_name, bottom_count, top_count);
            return -1;
        }
        mem += consumed;
        Layer* layer = LayerRegistry::CreateLayer(layer_type, rt_param);
        if (!layer) {
            LOGE("layer %s not exists or registered", layer_type);
            return FEATHER_ERR_UNSUPPORTED;  // net.cpp:107-111
        }
        layers[i] = layer;
        layer->name = std::string(layer_name);
        layer->type = std::string(layer_type);
        layer->bottoms.resize(bottom_count);
        for (int j = 0; j < bottom_count; j++) {
            char bottom_name[257];
            if (sscanf(mem, "%256s%n", bottom_name, &consumed) != 1) return -1;
            mem += consumed;
            std::map<std::string, Blob<float>*>::iterator it = blob_map.find(bottom_name);
            if (it == blob_map.end()) {
                LOGE("Topology error: bottom blob %s of layer %s type %s not found in map.", bottom_name, layer_name, layer_type);
                layer->bottoms.clear();
                return FEATHER_ERR_TOPOLOGY;  // net.cpp:127-131
            }
            layer->bottoms[j] = it->second;
        }
        layer->tops.resize(top_count);
        for (int j = 0; j < top_count; j++) {
            char top_name[257];
            if (sscanf(mem, "%256s%n", top_name, &consumed) != 1) return -1;
            mem += consumed;
            layer->tops[j] = new Blob<float>(top_name);
            blob_map[top_name] = layer->tops[j];
        }
        const int pdlr = pd.load_param_mem(mem);
        if (pdlr != 0) {
            LOGE("ParamDict load_param failed");
            return pdlr;
        }
        const int lr = layer->LoadParam(pd);
        if (lr != 0) {
            LOGE("Layer %s load_param failed", layer_name);
            return lr;
        }
        if (layer->type == "Input" && input_name_.empty() && !layer->tops.empty()) {
            input_name_ = layer->tops[0]->name;
            InputLayer* il = static_cast<InputLayer*>(layer);
            input_c_ = il->c; input_h_ = il->h; input_w_ = il->w;
        }
    }
    _param_loaded = 1;
    return 0;
}

int Net::LoadWeights(const char* path) {
    FILE* fp = fopen(path, "rb");
    if (fp == NULL) {
        LOGE("Cannot open weights file, path: %s", path);
        return -1;
    }
    const int rc = this->LoadWeights(fp);
    fclose(fp);
    return rc;
}

int Net::LoadWeightsFrom(const ncnn::ModelBin& mb, bool upload) {
    if (this->_net_initialized) {
        LOGE("Net is already initialized. Are you repeatedly loading models?");
        return -1;
    }
    if (this->layers.empty()) {
        LOGE("Network has not been loaded. Please load the param file first.");
        return -1;
    }
    for (size_t i = 0; i < this->layers.size(); i++) {
        Layer* layer = layers[i];
        if (!layer) {
            LOGE("LoadWeights error at layer %d, parameter file has inconsistent content.", (int)i);
            return -1;
        }
        const int lret = layer->LoadWeights(mb);
        if (lret != 0) {
            LOGE("Layer %s loading weights failed with exit code %d", layer->name.c_str(), lret);
            return -1;
        }
    }
    return BindWeightBlobs(upload);
}

int Net::LoadWeights(FILE* fp) {
    ncnn::ModelBinFromStdio mb(fp);
    const int rc = LoadWeightsFrom(mb, true);
    if (rc == 0) this->_weights_loaded = 1;
    return rc;
}

int Net::PrepareWeightArena() {
    ncnn::ModelBinSizesOnly mb;
    return LoadWeightsFrom(mb, false);
}

int Net::AttachWeights() {
    if (!weight_arena_ && weight_arena_floats_ > 0) return -1;
    this->_weights_loaded = 1;
    return 0;
}

// Lay every staged weight blob out in one device allocation (256-byte aligned slices), upload once.
int Net::BindWeightBlobs(bool upload) {
    std::vector<Blob<float>*> staged;
    size_t total = 0;
    std::vector<size_t> offsets;
    for (size_t i = 0; i < layers.size(); ++i)
        for (size_t j = 0; j < layers[i]->weights.size(); ++j) {
            Blob<float>* b = layers[i]->weights[j];
            if (!b->staged()) continue;
            staged.push_back(b);
            offsets.push_back(total);
            total += (b->data_size() + 63) & ~static_cast<size_t>(63);
        }
    if (weight_arena_) {
        cudaFree(weight_arena_);
        weight_arena_ = nullptr;
    }
    weight_arena_floats_ = total;
    if (total == 0) return 0;
    CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&weight_arena_), total * sizeof(float)));
    if (upload) {
        float* host = nullptr;
        CUDA_OK(cudaMallocHost(reinterpret_cast<void**>(&host), total * sizeof(float)));
        memset(host, 0, total * sizeof(float));
        for (size_t i = 0; i < staged.size(); ++i)
            memcpy(host + offsets[i], staged[i]->host_stage().data(), staged[i]->data_size() * sizeof(float));
        cudaError_t e = cudaMemcpy(weight_arena_, host, total * sizeof(float), cudaMemcpyHostToDevice);
        cudaFreeHost(host);
        CUDA_OK(e);
    }
    for (size_t i = 0; i < staged.size(); ++i) staged[i]->BindExternal(weight_arena_ + offsets[i]);
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// README-era loaders
// ---------------------------------------------------------------------------------------------------------
int Net::InitFromBuffer(const void* net_buffer, size_t size) {
    const unsigned char* p = static_cast<const unsigned char*>(net_buffer);
    if (size < 16 || memcmp(p, kContainerMagic, 8) != 0) {
        LOGE("not a .feathermodel container (magic FTHRB200 missing)");
        return -1;
    }
    uint64_t param_len = 0;
    memcpy(&param_len, p + 8, 8);
    if (param_len > size - 16) return -1;  // (16 + param_len > size would wrap for a huge param_len)
    std::string text(reinterpret_cast<const char*>(p + 16), static_cast<size_t>(param_len));
    int rc = ParseParamText(text.c_str());
    if (rc) return rc;
    const unsigned char* bin = p + 16 + param_len;
    ncnn::ModelBinFromMemory mb(bin, p + size);  // bounded: a truncated container fails like a short fread
    rc = LoadWeightsFrom(mb, true);
    if (rc == 0) _weights_loaded = 1;
    return rc;
}

// Graph only (no weights): what a non-root member of a NetGroup / a non-root rank needs before PrepareWeightArena.
int Net::InitGraphFromBuffer(const void* net_buffer, size_t size) {
    const unsigned char* p = static_cast<const unsigned char*>(net_buffer);
    if (size < 16 || memcmp(p, kContainerMagic, 8) != 0) {
        LOGE("not a .feathermodel container (magic FTHRB200 missing)");
        return -1;
    }
    uint64_t param_len = 0;
    memcpy(&param_len, p + 8, 8);
    if (param_len > size - 16) return -1;
    std::string text(reinterpret_cast<const char*>(p + 16), static_cast<size_t>(param_len));
    return ParseParamText(text.c_str());
}

int Net::InitFromFile(FILE* fp) {
    fseek(fp, 0, SEEK_END);
    const long len = ftell(fp);
    fseek(fp, 0, SEEK_SET);
    if (len <= 0) return -1;
    std::vector<unsigned char> buf(static_cast<size_t>(len));
    if (fread(buf.data(), 1, buf.size(), fp) != buf.size()) return -1;
    return InitFromBuffer(buf.data(), buf.size());
}

int Net::InitFromPath(const char* model_path) {
    FILE* fp = fopen(model_path, "rb");
    if (fp) {
        char magic[8] = {0};
        const size_t got = fread(magic, 1, 8, fp);
        if (got == 8 && memcmp(magic, kContainerMagic, 8) == 0) {
            const int rc = InitFromFile(fp);
            fclose(fp);
            return rc;
        }
        fclose(fp);
    }
    const std::string base(model_path);
    int rc = LoadParam((base + ".param").c_str());
    if (rc) return rc;
    return LoadWeights((base + ".bin").c_str());
}

// ---------------------------------------------------------------------------------------------------------
// Input / output
// ---------------------------------------------------------------------------------------------------------
int Net::FeedInput(const char* input_name, ncnn::Mat& in) {
    std::map<std::string, Blob<float>*>::iterator it = this->blob_map.find(std::string(input_name));
    if (it == blob_map.end()) {
        LOGE("Invalid input blob %s, not found in map.", input_name);
        return -1;
    }
    return it->second->CopyFromMat(in);
}

int Net::FeedInputBatch(const char* input_name, const float* host_nchw, int n, int c, int h, int w) {
    std::map<std::string, Blob<float>*>::iterator it = this->blob_map.find(std::string(input_name));
    if (it == blob_map.end() || !host_nchw || n < 1) return -1;
    it->second->ReshapeWithRealloc(n, c, h, w);
    return it->second->CopyFromHost(host_nchw, rt_param->stream());
}

// ncnn::Mat::from_pixels[_resize] + substract_mean_normalize + FeedInput (README.md:64-66 usage), for a whole batch and on
// the device: the u8 images cross PCIe (4x fewer bytes than fp32) and one fused kernel writes the input blob.
int Net::FeedInputPixels(const char* input_name, const unsigned char* host_pixels, int type, int w, int h, int target_w,
                         int target_h, int batch, const float* mean_vals, const float* norm_vals) {
    std::map<std::string, Blob<float>*>::iterator it = this->blob_map.find(std::string(input_name));
    if (it == blob_map.end() || !host_pixels || batch < 1) return -1;
    int src_c = 0, out_c = 0;
    int rc = fcuda_pixel_channels(type, &src_c, &out_c);
    if (rc) return rc;
    if (target_w <= 0) target_w = w;
    if (target_h <= 0) target_h = h;
    const size_t bytes = static_cast<size_t>(batch) * w * h * src_c;
    cudaStream_t s = static_cast<cudaStream_t>(rt_param->stream());
    if (bytes > pixel_stage_bytes_) {
        if (pixel_stage_) {
            CUDA_OK(cudaStreamSynchronize(s));
            cudaFree(pixel_stage_);
        }
        pixel_stage_ = nullptr;
        pixel_stage_bytes_ = 0;
        CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&pixel_stage_), bytes));
        pixel_stage_bytes_ = bytes;
    }
    CUDA_OK(cudaMemcpyAsync(pixel_stage_, host_pixels, bytes, cudaMemcpyHostToDevice, s));
    it->second->ReshapeWithRealloc(batch, out_c, target_h, target_w);
    if (!it->second->data()) return FEATHER_ERR_CUDA;
    return fcuda_from_pixels(it->second->data(), pixel_stage_, type, w, h, target_w, target_h, mean_vals, norm_vals, batch, s);
}

int Net::FeedInputDevice(const char* input_name, const float* device_nchw, int n, int c, int h, int w) {
    std::map<std::string, Blob<float>*>::iterator it = this->blob_map.find(std::string(input_name));
    if (it == blob_map.end() || !device_nchw || n < 1) return -1;
    it->second->ViewExternal(const_cast<float*>(device_nchw), n, c, h, w);
    return 0;
}

int Net::ForwardBatch(const float* host_nchw, int batch) {
    if (input_name_.empty() || input_c_ <= 0) return -1;
    int rc = FeedInputBatch(input_name_.c_str(), host_nchw, batch, input_c_, input_h_, input_w_);
    if (rc) return rc;
    return Forward();
}

int Net::Forward(const float* input) { return ForwardBatch(input, 1); }

int Net::Forward(const float* input, int height, int width) {
    if (input_name_.empty() || input_c_ <= 0) return -1;
    int rc = FeedInputBatch(input_name_.c_str(), input, 1, input_c_, height, width);
    if (rc) return rc;
    return Forward();
}

int Net::Synchronize() {
    CUDA_OK(cudaStreamSynchronize(static_cast<cudaStream_t>(rt_param->stream())));
    return 0;
}

int Net::ExtractDevice(std::string name, const float** device_ptr, int* n, int* c, int* h, int* w) {
    std::map<std::string, Blob<float>*>::iterator it = blob_map.find(name);
    if (it == blob_map.end()) {
        LOGE("Cannot find output blob %s", name.c_str());
        return -1;
    }
    const Blob<float>* p_blob = it->second;
    if (!p_blob->data()) return -1;  // fused away or never produced
    *device_ptr = p_blob->data();
    if (n) *n = p_blob->num();
    if (c) *c = p_blob->channels();
    if (h) *h = p_blob->height();
    if (w) *w = p_blob->width();
    return 0;
}

int Net::Extract(std::string name, float** output_ptr, int* n, int* c, int* h, int* w) {
    const float* dptr = NULL;
    int rc = ExtractDevice(name, &dptr, n, c, h, w);
    if (rc) return rc;
    const Blob<float>* p_blob = blob_map[name];
    std::vector<float>& mirror = host_mirror_[name];
    mirror.resize(p_blob->data_size());
    rc = p_blob->CopyToHost(mirror.data(), rt_param->stream());
    if (rc) return rc;
    *output_ptr = mirror.data();
    return 0;
}

int Net::Extract(std::string blob_name, ncnn::Mat& out) {
    float* data = NULL;
    int n, c, h, w;
    int rc = Extract(blob_name, &data, &n, &c, &h, &w);
    if (rc) return rc;
    const int rank = blob_map[blob_name]->dims();
    if (rank == 1 || rank == 2) {  // ncnn Mat(w) / Mat(w, h): dense, no channel step
        if (rank == 1) out.create(w, static_cast<size_t>(4));
        else out.create(w, h, static_cast<size_t>(4));
        memcpy(out.data, data, sizeof(float) * static_cast<size_t>(w) * h);
        return 0;
    }
    out.create(w, h, c, 4U);
    const size_t stride = static_cast<size_t>(w) * h;
    for (int ch = 0; ch < c; ++ch) memcpy(out.channel(ch).data, data + stride * ch, sizeof(float) * stride);
    return 0;
}

int Net::ExtractBlob(float* output_ptr, std::string blob_name) {
    std::map<std::string, Blob<float>*>::iterator it = blob_map.find(blob_name);
    if (it == blob_map.end() || !it->second->data()) {
        LOGE("Cannot find output blob %s", blob_name.c_str());
        return -1;
    }
    return it->second->CopyToHost(output_ptr, rt_param->stream());
}

int Net::GetBlobDataSize(size_t* data_size, std::string blob_name) {
    std::map<std::string, Blob<float>*>::iterator it = blob_map.find(blob_name);
    if (it == blob_map.end()) {
        LOGE("Cannot find output blob %s", blob_name.c_str());
        return -1;
    }
    *data_size = it->second->data_size();
    return 0;
}

std::vector<std::string> Net::BlobNames() const {
    std::vector<std::string> names;
    for (std::map<std::string, Blob<float>*>::const_iterator it = blob_map.begin(); it != blob_map.end(); ++it)
        names.push_back(it->first);
    return names;
}

int Net::BuildBlobMap() {
    blob_map.clear();
    for (size_t i = 0; i < layers.size(); ++i)
        for (size_t j = 0; j < layers[i]->tops.size(); ++j) blob_map[layers[i]->tops[j]->name] = layers[i]->tops[j];
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Forward
// ---------------------------------------------------------------------------------------------------------
int Net::Reshape() {
    // MemoryData holds one copy per image of the batch the first Input was fed
    int batch = 1;
    std::map<std::string, Blob<float>*>::iterator in = blob_map.find(input_name_);
    if (in != blob_map.end() && in->second->num() > 0) batch = static_cast<int>(in->second->num());
    for (size_t i = 0; i < layers.size(); ++i) {
        Layer* layer = layers[i];
        if (layer->_fused_away) continue;
        if (MemoryDataLayer* md = dynamic_cast<MemoryDataLayer*>(layer)) md->set_batch(batch);
        const int gr = layer->Reshape();
        if (gr != 0) {
            LOGE("Layer %s failed to generate tops (%d)", layer->name.c_str(), gr);
            return FEATHER_ERR_WEIGHTS;  // net.cpp:250-254
        }
    }
    return 0;
}

int Net::InitLayers() {
    for (size_t i = 0; i < layers.size(); ++i) {
        if (layers[i]->_fused_away) continue;
        const int rc = layers[i]->Init();
        if (rc != 0) {
            LOGE("Layer %s failed to initialise (%d)", layers[i]->name.c_str(), rc);
            return rc;
        }
    }
    return 0;
}

int Net::RunLayers() {
    for (size_t i = 0; i < layers.size(); ++i) {
        if (layers[i]->_fused_away) continue;
        const int rc = layers[i]->Forward();  // unlike the reference (net.cpp:318) return codes are checked
        if (rc != 0) {
            LOGE("Layer %s type %s Forward failed (%d)", layers[i]->name.c_str(), layers[i]->type.c_str(), rc);
            return rc;
        }
    }
    return 0;
}

// A two-input sum the residual and super-resolution tail passes may absorb: a plain Eltwise SUM (Caffe's layout), or a
// BinaryOp ADD of two bottoms without a scalar (how onnx2ncnn and pnnx write the same add).  *relu gets the ReLU it has
// absorbed; *broadcast whether its addends may broadcast (BinaryOp), which Reshape of the absorbing layer then checks.
static bool two_input_sum(Layer* l, int* relu, bool* broadcast) {
    if (l->_fused_away || l->bottoms.size() != 2 || l->tops.size() != 1) return false;
    if (const EltwiseLayer* e = dynamic_cast<const EltwiseLayer*>(l)) {
        *relu = e->fused_relu();
        *broadcast = false;
        return e->plain_sum();
    }
    if (const BinaryOpLayer* b = dynamic_cast<const BinaryOpLayer*>(l)) {
        *relu = b->fused_relu();
        *broadcast = true;
        return b->plain_add();
    }
    return false;
}

// The live version of the reference's dead TryFuse/Fuse hooks (layer.h:61-68, SURVEY.md §8f rank 1):
// a fusible producer absorbs its consumer when that consumer is the only reader of the producer's top.
int Net::ApplyFusion() {
    std::map<Blob<float>*, int> readers;
    for (size_t i = 0; i < layers.size(); ++i)
        for (size_t j = 0; j < layers[i]->bottoms.size(); ++j) readers[layers[i]->bottoms[j]]++;
    for (size_t i = 0; i < layers.size(); ++i) {
        Layer* a = layers[i];
        if (a->_fused_away || !a->fusible() || a->tops.size() != 1) continue;
        for (size_t j = i + 1; j < layers.size(); ++j) {
            Layer* b = layers[j];
            if (b->_fused_away) continue;
            if (b->bottoms.size() != 1 || b->tops.size() != 1 || b->bottoms[0] != a->tops[0]) break;
            if (readers[a->tops[0]] != 1) break;
            if (a->TryFuse(b) != 1) break;
            // a now produces b's top; a's former top is never materialised
            Blob<float>* dead = a->tops[0];
            blob_map.erase(dead->name);
            delete dead;
            a->tops[0] = b->tops[0];
            b->tops.clear();
            b->bottoms.clear();
            b->_fused_away = true;
        }
    }
    // Second pass: a two-input sum (two_input_sum, +ReLU absorbed above) whose one addend is a convolution's otherwise
    // unread top becomes that convolution's epilogue (ResNet shortcuts: 16 add_relu passes over the activations in
    // ResNet-50).  The other addend must already exist when the convolution runs.
    std::map<Blob<float>*, size_t> producer;
    for (size_t i = 0; i < layers.size(); ++i)
        for (size_t j = 0; j < layers[i]->tops.size(); ++j) producer[layers[i]->tops[j]] = i;
    for (size_t j = 0; j < layers.size(); ++j) {
        Layer* e = layers[j];
        int relu = 0;
        bool broadcast = false;
        if (!two_input_sum(e, &relu, &broadcast)) continue;
        for (int k = 1; k >= 0; --k) {
            Blob<float>* mine = e->bottoms[k];
            Blob<float>* other = e->bottoms[1 - k];
            if (mine == other || readers[mine] != 1 || !producer.count(mine)) continue;
            const size_t i = producer[mine];
            ConvLayer* conv = dynamic_cast<ConvLayer*>(layers[i]);
            if (!conv || i >= j || conv->_fused_away || conv->tops.size() != 1) continue;
            if (producer.count(other) && producer[other] >= i) continue;  // not computed yet when the conv runs
            if (conv->param().activation != booster::None) continue;      // its own ReLU would have to precede the sum
            if (conv->FuseResidual(other, relu, broadcast) != 1) continue;
            Blob<float>* dead = conv->tops[0];
            blob_map.erase(dead->name);
            producer.erase(dead);
            delete dead;
            conv->tops[0] = e->tops[0];
            producer[conv->tops[0]] = i;
            e->tops.clear();
            e->bottoms.clear();
            e->_fused_away = true;
            break;
        }
    }
    // Third pass: a Crop of a deconvolution's otherwise unread top becomes part of the deconvolution's pads (FCN's final
    // crop of the upsampled scores to the input size: one full read and write of the largest blob fewer).  Like the
    // residual addend, the Crop's reference blob must already exist when the deconvolution runs.
    for (size_t j = 0; j < layers.size(); ++j) {
        CropLayer* c = dynamic_cast<CropLayer*>(layers[j]);
        if (!c || c->_fused_away || c->bottoms.empty() || c->tops.size() != 1) continue;
        Blob<float>* mine = c->bottoms[0];
        Blob<float>* ref = c->reference();
        if (mine == ref || readers[mine] != 1 || !producer.count(mine)) continue;
        const size_t i = producer[mine];
        DeconvLayer* d = dynamic_cast<DeconvLayer*>(layers[i]);
        if (!d || i >= j || d->_fused_away || d->tops.size() != 1) continue;
        if (ref && producer.count(ref) && producer[ref] >= i) continue;  // not computed yet when the deconvolution runs
        if (d->FoldCrop(c->window(), ref) != 1) continue;
        Blob<float>* dead = d->tops[0];
        blob_map.erase(dead->name);
        producer.erase(dead);
        delete dead;
        d->tops[0] = c->tops[0];
        producer[d->tops[0]] = i;
        c->tops.clear();
        c->bottoms.clear();
        c->_fused_away = true;
    }
    // Super-resolution tail pass (ahead of the routing pass, which ends early when its tuning switch is off): a
    // two-input sum (two_input_sum) without a ReLU of a PixelShuffle's top and a nearest Interp's top, each read only by
    // the sum, becomes the PixelShuffle's tail (SRVGGNetCompact's out = pixel_shuffle(conv) + nearest_upsample(x): two
    // full-size blobs neither written nor read back).  Like the residual addend, the Interp's input must already exist
    // when the PixelShuffle runs.  PixelShuffleLayer::Reshape rejects a tail whose addends do not have one shape.
    for (size_t j = 0; j < layers.size(); ++j) {
        Layer* e = layers[j];
        int relu = 0;
        bool broadcast = false;
        if (!two_input_sum(e, &relu, &broadcast) || relu) continue;
        for (int k = 0; k < 2; ++k) {
            Blob<float>* mine = e->bottoms[k];
            Blob<float>* other = e->bottoms[1 - k];
            if (mine == other || readers[mine] != 1 || readers[other] != 1 || !producer.count(mine) ||
                !producer.count(other))
                continue;
            const size_t i = producer[mine], m = producer[other];
            PixelShuffleLayer* ps = dynamic_cast<PixelShuffleLayer*>(layers[i]);
            InterpLayer* up = dynamic_cast<InterpLayer*>(layers[m]);
            if (!ps || !up || i >= j || m >= j || ps->_fused_away || up->_fused_away || ps->tops.size() != 1 ||
                up->tops.size() != 1 || up->bottoms.size() != 1)
                continue;
            Blob<float>* base = up->bottoms[0];
            if (producer.count(base) && producer[base] >= i) continue;  // not computed yet when the PixelShuffle runs
            if (ps->FuseUpsampledAdd(up->interp_param(), base) != 1) continue;
            for (Blob<float>* dead : {mine, other}) {
                blob_map.erase(dead->name);
                producer.erase(dead);
                delete dead;
            }
            ps->tops[0] = e->tops[0];
            producer[ps->tops[0]] = i;
            up->tops.clear();
            up->bottoms.clear();
            up->_fused_away = true;
            e->tops.clear();
            e->bottoms.clear();
            e->_fused_away = true;
            break;
        }
    }
    // Fourth pass: channel routing.  Concat (axis 0) -> ShuffleChannel -> Slice (axis 0), or any two adjacent of them,
    // run as one fcuda_route_forward launch by the chain's last layer (ShuffleNet-v2 units: one read and one write of
    // the activation instead of three of each).  Every intermediate blob must have that layer as its only reader.  A
    // layer absorbs its producer's bottoms, so a ShuffleChannel that took a Concat passes both on to a Slice.
    if (fcuda_get_tuning("route_fuse") != 1) return 0;
    std::map<Blob<float>*, Layer*> made_by;
    for (size_t i = 0; i < layers.size(); ++i)
        for (size_t j = 0; j < layers[i]->tops.size(); ++j) made_by[layers[i]->tops[j]] = layers[i];
    for (size_t j = 0; j < layers.size(); ++j) {
        RouteLayer* r = dynamic_cast<RouteLayer*>(layers[j]);
        if (!r || r->_fused_away || r->absorbed() || r->bottoms.size() != 1) continue;
        SliceLayer* slice = dynamic_cast<SliceLayer*>(r);
        if (slice && slice->axis() != 0) continue;
        Blob<float>* mine = r->bottoms[0];
        if (readers[mine] != 1 || !made_by.count(mine)) continue;
        Layer* p = made_by[mine];
        if (p->_fused_away || p->tops.size() != 1) continue;
        ConcatLayer* cat = dynamic_cast<ConcatLayer*>(p);
        ShuffleChannelLayer* sh = slice ? dynamic_cast<ShuffleChannelLayer*>(p) : nullptr;
        if (cat && (cat->param_axis() != 0 || cat->bottoms.empty() || cat->bottoms.size() > FCUDA_ROUTE_MAX)) continue;
        if (!cat && !sh) continue;
        r->Absorb(p->bottoms, sh != nullptr, sh ? sh->group() : 1, sh ? sh->reverse() : 0);
        blob_map.erase(mine->name);
        delete mine;
        p->tops.clear();
        p->bottoms.clear();
        p->_fused_away = true;
    }
    return 0;
}

int Net::FuseNow() {
    if (!_param_loaded) return -1;
    if (fusion_ && !fusion_applied_) {
        ApplyFusion();
        fusion_applied_ = true;
    }
    int n = 0;
    for (size_t i = 0; i < layers.size(); ++i) n += layers[i]->_fused_away ? 1 : 0;
    return n;
}

int Net::LayerFusedAway(const std::string& layer_name) const {
    for (size_t i = 0; i < layers.size(); ++i)
        if (layers[i]->name == layer_name) return layers[i]->_fused_away ? 1 : 0;
    return -1;
}

int Net::LayerConvAlgo(const std::string& layer_name) const {
    for (size_t i = 0; i < layers.size(); ++i) {
        if (layers[i]->name != layer_name) continue;
        const ConvLayer* conv = dynamic_cast<const ConvLayer*>(layers[i]);
        return (conv && !conv->_fused_away) ? conv->algo() : -1;
    }
    return -1;
}

void Net::ResetGraph() {
    for (auto& kv : graph_cache_) cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(kv.second));
    graph_cache_.clear();
    warmed_keys_.clear();
}

int Net::Forward() {
    if (!_param_loaded || !_weights_loaded) {
        LOGE("Forward called before the model was loaded");
        return -1;
    }
    if (fusion_ && !fusion_applied_) {
        ApplyFusion();
        fusion_applied_ = true;
    }
    int rc = this->Reshape();
    if (rc) return rc;
    // Packed filters are laid out for the precision mode (1 or 2 operand planes) that was current at Init: a later
    // fcuda_set_precision() must re-pack them before any kernel reads `packed + plane` (ADVICE r1).
    const int precision_now = fcuda_get_precision();
    if (this->_net_initialized == 0 || precision_now != init_precision_) {
        if (this->_net_initialized) ResetGraph();
        rc = InitLayers();
        if (rc) return rc;
        this->_net_initialized = 1;
        init_precision_ = precision_now;
    }
    cudaStream_t s = static_cast<cudaStream_t>(rt_param->stream());

    // The scratch pool is sized by Reshape (Request) and must exist BEFORE a stream capture begins: cudaMalloc /
    // cudaFree are illegal inside one.  A pool that moved invalidates every captured graph (they hold its address).
    {
        CommonMemPool<float>* pool = rt_param->common_mempool();
        if (!pool->Alloc()) return FEATHER_ERR_CUDA;
        float* pool_ptr = nullptr;
        pool->GetPtr(&pool_ptr);
        if (pool_ptr != graph_pool_ptr_) {
            ResetGraph();
            graph_pool_ptr_ = pool_ptr;
        }
    }

    // CUDA-graph replay: one instantiated graph per (blob addresses, blob shapes, scratch pool, precision) key, so
    // rotating between a few input buffers / batch sizes replays without re-capturing.  Shapes are part of the key:
    // blobs are grow-only, so two geometries with equal element counts share addresses (224x112 vs 112x224).
    std::vector<size_t> key;
    if (use_graph_ && s != nullptr) {
        key.push_back(reinterpret_cast<size_t>(graph_pool_ptr_));
        key.push_back(static_cast<size_t>(precision_now));
        for (size_t i = 0; i < layers.size(); ++i)
            for (size_t j = 0; j < layers[i]->tops.size(); ++j) {
                const Blob<float>* b = layers[i]->tops[j];
                key.push_back(reinterpret_cast<size_t>(b->data()));
                key.push_back((b->num() << 40) ^ (b->channels() << 20) ^ b->height());
                key.push_back(b->width());
            }
        std::map<std::vector<size_t>, void*>::iterator hit = graph_cache_.find(key);
        if (hit != graph_cache_.end()) {
            CUDA_OK(cudaGraphLaunch(static_cast<cudaGraphExec_t>(hit->second), s));
            return 0;
        }
    }

    const unsigned long long before = fcuda_launch_count();
    // The first Forward of every new key runs eagerly (kernel attributes, lazily created tensor maps); the second one
    // with that key is captured.
    if (use_graph_ && s != nullptr && warmed_keys_.count(key)) {
        if (graph_cache_.size() >= 16) ResetGraph();
        cudaGraph_t graph = nullptr;
        CUDA_OK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        rc = RunLayers();
        cudaError_t e = cudaStreamEndCapture(s, &graph);
        if (rc != 0 || e != cudaSuccess) {
            if (graph) cudaGraphDestroy(graph);
            LOGE("CUDA graph capture failed (%d, %s); running eagerly", rc, cudaGetErrorString(e));
            cudaGetLastError();
            use_graph_ = false;
            return RunLayers();
        }
        cudaGraphExec_t exec = nullptr;
        e = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        CUDA_OK(e);
        graph_cache_[key] = exec;
        launches_per_forward_ = fcuda_launch_count() - before;
        CUDA_OK(cudaGraphLaunch(exec, s));
        return 0;
    }
    rc = RunLayers();
    launches_per_forward_ = fcuda_launch_count() - before;
    if (use_graph_ && s != nullptr && rc == 0) {
        if (warmed_keys_.size() >= 64) warmed_keys_.clear();
        warmed_keys_.insert(key);
    }
    return rc;
}

// ---------------------------------------------------------------------------------------------------------
// Pipelined end-to-end path: host batch -> H2D (copy stream) -> Forward -> D2H of one blob, two batches in flight.
// The H2D copy of batch i+1 runs behind an event while batch i computes; what FeedInput (net.cpp:232-243) does
// synchronously per image in the reference.
// ---------------------------------------------------------------------------------------------------------
int Net::SubmitBatch(const float* host_nchw, int batch, const char* blob_name, float* host_out) {
    if (input_name_.empty() || input_c_ <= 0 || !host_nchw || batch < 1) return -1;
    cudaStream_t s = static_cast<cudaStream_t>(rt_param->stream());
    if (!copy_stream_) {
        cudaStream_t cs = nullptr;
        CUDA_OK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        copy_stream_ = cs;
    }
    cudaStream_t cs = static_cast<cudaStream_t>(copy_stream_);
    PipeSlot& sl = pipe_[submitted_ & 1];
    if (!sl.ev_h2d) {
        cudaEvent_t a, b, c;
        CUDA_OK(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
        CUDA_OK(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
        CUDA_OK(cudaEventCreateWithFlags(&c, cudaEventDisableTiming));
        sl.ev_h2d = a; sl.ev_free = b; sl.ev_done = c;
    }
    const size_t floats = static_cast<size_t>(batch) * input_c_ * input_h_ * input_w_;
    if (floats > sl.capacity) {
        if (sl.used) CUDA_OK(cudaEventSynchronize(static_cast<cudaEvent_t>(sl.ev_done)));
        if (sl.dev) cudaFree(sl.dev);
        sl.dev = nullptr;
        sl.capacity = 0;
        CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&sl.dev), floats * sizeof(float)));
        sl.capacity = floats;
    }
    // the previous Forward that read this slot must have finished before the slot is overwritten
    if (sl.used) CUDA_OK(cudaStreamWaitEvent(cs, static_cast<cudaEvent_t>(sl.ev_free), 0));
    CUDA_OK(cudaMemcpyAsync(sl.dev, host_nchw, floats * sizeof(float), cudaMemcpyHostToDevice, cs));
    CUDA_OK(cudaEventRecord(static_cast<cudaEvent_t>(sl.ev_h2d), cs));
    CUDA_OK(cudaStreamWaitEvent(s, static_cast<cudaEvent_t>(sl.ev_h2d), 0));
    int rc = FeedInputDevice(input_name_.c_str(), sl.dev, batch, input_c_, input_h_, input_w_);
    if (rc) return rc;
    rc = Forward();
    if (rc) return rc;
    CUDA_OK(cudaEventRecord(static_cast<cudaEvent_t>(sl.ev_free), s));
    if (blob_name && host_out) {
        std::map<std::string, Blob<float>*>::iterator it = blob_map.find(blob_name);
        if (it == blob_map.end() || !it->second->data()) return -1;
        CUDA_OK(cudaMemcpyAsync(host_out, it->second->data(), it->second->data_size() * sizeof(float),
                                cudaMemcpyDeviceToHost, s));
    }
    CUDA_OK(cudaEventRecord(static_cast<cudaEvent_t>(sl.ev_done), s));
    sl.used = true;
    return static_cast<int>(submitted_++ & 0x3fffffff);
}

int Net::WaitBatch(int ticket) {
    if (ticket < 0) return -1;
    PipeSlot& sl = pipe_[ticket & 1];
    if (!sl.used) return -1;
    CUDA_OK(cudaEventSynchronize(static_cast<cudaEvent_t>(sl.ev_done)));
    return 0;
}

void Net::FreePipeline() {
    for (int i = 0; i < 2; ++i) {
        PipeSlot& sl = pipe_[i];
        if (sl.ev_h2d) cudaEventDestroy(static_cast<cudaEvent_t>(sl.ev_h2d));
        if (sl.ev_free) cudaEventDestroy(static_cast<cudaEvent_t>(sl.ev_free));
        if (sl.ev_done) cudaEventDestroy(static_cast<cudaEvent_t>(sl.ev_done));
        if (sl.dev) cudaFree(sl.dev);
        sl = PipeSlot();
    }
    if (copy_stream_) cudaStreamDestroy(static_cast<cudaStream_t>(copy_stream_));
    copy_stream_ = nullptr;
}

}  // inline namespace b200
}  // namespace feather

inline namespace feather_b200 {
int ChkParamHeader(FILE* fp) {
    fseek(fp, 0, SEEK_SET);
    int magic = 0;
    if (fscanf(fp, "%d", &magic) != 1) {
        fprintf(stderr, "issue with param file\n");
        return -1;
    }
    if (magic != 7767517) {
        fprintf(stderr, "param is too old, please regenerate\n");
        return -1;
    }
    return 0;
}
}  // inline namespace feather_b200
