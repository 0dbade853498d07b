// extern "C" face of feather::Net for language bindings (ctypes in feathercnn_b200/net.py).
// Declared in include/feather_c.h.
#include <feather_c.h>

#include <feather/ncnn/modelbin.h>
#include <feather/net.h>
#include <feather/net_group.h>
#include <string.h>

#include <stdio.h>

#include <exception>
#include <string>

using feather::Net;
using feather::NetGroup;

// No C++ exception may cross the C boundary (a corrupt model must produce an error code, not std::terminate).
#define FNET_GUARD(expr)                                   \
    try {                                                  \
        return (expr);                                     \
    } catch (const std::exception& e) {                    \
        fprintf(stderr, "feather: %s\n", e.what());        \
        return FEATHER_ERR_WEIGHTS;                        \
    } catch (...) {                                        \
        return FEATHER_ERR_WEIGHTS;                        \
    }

extern "C" {

void* fnet_create(void) { return new Net(); }
void fnet_destroy(void* h) { delete static_cast<Net*>(h); }
void fnet_set_fusion(void* h, int enable) { static_cast<Net*>(h)->SetFusion(enable != 0); }
void fnet_set_cuda_graph(void* h, int enable) { static_cast<Net*>(h)->SetCudaGraph(enable != 0); }
long fnet_modelbin_load_mem(const unsigned char* buf, int w, int type, float* out) {
    const unsigned char* mem = buf;
    ncnn::ModelBinFromMemory mb(mem);
    ncnn::Mat m = mb.load(w, type);
    if (m.empty() || !out) return -1;
    memcpy(out, m.data, sizeof(float) * static_cast<size_t>(w));
    return static_cast<long>(mem - buf);
}
int fnet_fuse_now(void* h) { return static_cast<Net*>(h)->FuseNow(); }
int fnet_layer_fused_away(void* h, const char* name) { return static_cast<Net*>(h)->LayerFusedAway(name ? name : ""); }
int fnet_layer_conv_algo(void* h, const char* name) { return static_cast<Net*>(h)->LayerConvAlgo(name ? name : ""); }
void fnet_set_stream(void* h, void* stream) { static_cast<Net*>(h)->SetStream(stream); }
int fnet_load_param(void* h, const char* path) { FNET_GUARD(static_cast<Net*>(h)->LoadParam(path)) }
int fnet_load_param_text(void* h, const char* text) { FNET_GUARD(static_cast<Net*>(h)->LoadParamFromText(text)) }
int fnet_load_weights(void* h, const char* path) { FNET_GUARD(static_cast<Net*>(h)->LoadWeights(path)) }
int fnet_init_from_path(void* h, const char* path) { FNET_GUARD(static_cast<Net*>(h)->InitFromPath(path)) }
int fnet_init_from_buffer(void* h, const void* buf, size_t size) { FNET_GUARD(static_cast<Net*>(h)->InitFromBuffer(buf, size)) }
int fnet_prepare_weight_arena(void* h) { return static_cast<Net*>(h)->PrepareWeightArena(); }
int fnet_weight_arena(void* h, float** device_ptr, size_t* floats) {
    Net* n = static_cast<Net*>(h);
    *device_ptr = n->WeightArena();
    *floats = n->WeightArenaFloats();
    return 0;
}
int fnet_attach_weights(void* h) { return static_cast<Net*>(h)->AttachWeights(); }
int fnet_feed_input_batch(void* h, const char* name, const float* host, int n, int c, int hh, int w) {
    return static_cast<Net*>(h)->FeedInputBatch(name, host, n, c, hh, w);
}
int fnet_feed_input_pixels(void* h, const char* name, const unsigned char* host_pixels, int type, int w, int hh, int target_w,
                           int target_h, int batch, const float* mean_vals, const float* norm_vals) {
    FNET_GUARD(static_cast<Net*>(h)->FeedInputPixels(name, host_pixels, type, w, hh, target_w, target_h, batch, mean_vals, norm_vals))
}
int fnet_feed_input_device(void* h, const char* name, const float* dev, int n, int c, int hh, int w) {
    return static_cast<Net*>(h)->FeedInputDevice(name, dev, n, c, hh, w);
}
int fnet_forward(void* h) { FNET_GUARD(static_cast<Net*>(h)->Forward()) }
int fnet_forward_batch(void* h, const float* host_nchw, int batch) { FNET_GUARD(static_cast<Net*>(h)->ForwardBatch(host_nchw, batch)) }
int fnet_submit_batch(void* h, const float* host_nchw, int batch, const char* blob, float* host_out) {
    FNET_GUARD(static_cast<Net*>(h)->SubmitBatch(host_nchw, batch, blob, host_out))
}
int fnet_wait_batch(void* h, int ticket) { return static_cast<Net*>(h)->WaitBatch(ticket); }
int fnet_synchronize(void* h) { return static_cast<Net*>(h)->Synchronize(); }
int fnet_blob_shape(void* h, const char* name, int* n, int* c, int* hh, int* w) {
    Net* net = static_cast<Net*>(h);
    std::map<std::string, feather::Blob<float>*>::iterator it = net->blob_map.find(name);
    if (it == net->blob_map.end()) return -1;
    *n = it->second->num(); *c = it->second->channels(); *hh = it->second->height(); *w = it->second->width();
    return 0;
}
int fnet_blob_dims(void* h, const char* name) {
    Net* net = static_cast<Net*>(h);
    std::map<std::string, feather::Blob<float>*>::iterator it = net->blob_map.find(name);
    return it == net->blob_map.end() ? -1 : it->second->dims();
}
int fnet_extract_blob(void* h, const char* name, float* host_out) { return static_cast<Net*>(h)->ExtractBlob(host_out, name); }
int fnet_extract_device(void* h, const char* name, const float** dev, int* n, int* c, int* hh, int* w) {
    return static_cast<Net*>(h)->ExtractDevice(name, dev, n, c, hh, w);
}
unsigned long long fnet_launches_per_forward(void* h) { return static_cast<Net*>(h)->LaunchesPerForward(); }
int fnet_input_shape(void* h, int* c, int* hh, int* w) {
    static_cast<Net*>(h)->InputShape(c, hh, w);
    return 0;
}
// Writes the blob names separated by '\n' into buf (NUL terminated); returns the length needed.
size_t fnet_blob_names(void* h, char* buf, size_t cap) {
    std::string joined;
    for (const std::string& s : static_cast<Net*>(h)->BlobNames()) {
        if (!joined.empty()) joined += '\n';
        joined += s;
    }
    if (buf && cap > 0) {
        const size_t n = joined.size() < cap - 1 ? joined.size() : cap - 1;
        memcpy(buf, joined.data(), n);
        buf[n] = '\0';
    }
    return joined.size() + 1;
}
const char* fnet_input_name(void* h) { return static_cast<Net*>(h)->InputName().c_str(); }


// ---- feather::NetGroup (include/feather/net_group.h): one model on several GPUs of one box from one process --------------
void* fgroup_create(void) { return new NetGroup(); }
void fgroup_destroy(void* g) { delete static_cast<NetGroup*>(g); }
void fgroup_set_options(void* g, int fusion, int cuda_graph) {
    static_cast<NetGroup*>(g)->SetFusion(fusion != 0);
    static_cast<NetGroup*>(g)->SetCudaGraph(cuda_graph != 0);
}
int fgroup_init_from_path(void* g, const char* model_path, const int* devices, int count) {
    FNET_GUARD(static_cast<NetGroup*>(g)->InitFromPath(model_path, devices, count))
}
int fgroup_size(void* g) { return static_cast<NetGroup*>(g)->Size(); }
int fgroup_device(void* g, int i) {
    NetGroup* grp = static_cast<NetGroup*>(g);
    return (i >= 0 && i < grp->Size()) ? grp->Device(i) : -1;
}
void* fgroup_member(void* g, int i) {
    NetGroup* grp = static_cast<NetGroup*>(g);
    return (i >= 0 && i < grp->Size()) ? grp->Member(i) : nullptr;
}
const char* fgroup_broadcast_transport(void* g) { return static_cast<NetGroup*>(g)->BroadcastTransport(); }
int fgroup_forward_batch(void* g, const float* host_nchw, int batch, const char* blob, float* host_out) {
    FNET_GUARD(static_cast<NetGroup*>(g)->ForwardBatch(host_nchw, batch, blob, host_out))
}
int fgroup_shard_range(int batch, int members, int i, int* lo, int* hi) {
    if (!lo || !hi || members < 1 || i < 0 || i >= members || batch < 0) return -1;
    NetGroup::ShardRange(batch, members, i, lo, hi);
    return 0;
}
int fgroup_synchronize(void* g) { return static_cast<NetGroup*>(g)->Synchronize(); }
}  // extern "C"
