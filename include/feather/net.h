// feather::Net — the user-facing inference API.
//
// Keeps the surface of the reference snapshot (/root/reference/src/net.h:30-70: LoadParam / LoadWeights /
// FeedInput / Forward / Extract on ncnn .param/.bin models) and the README-era names the north star asks for
// (/root/reference/README.md:56-75: Net(num_threads), InitFromPath, Forward(float*), ExtractBlob,
// GetBlobDataSize), and adds what a GPU engine needs: a batch dimension, device-resident blobs, a CUDA stream,
// a contiguous device weight arena (one upload / one NCCL broadcast per model) and CUDA-graph replay.
//
// `.feathermodel`: the upstream flatbuffers schema is absent from the reference snapshot (SURVEY.md §0.1),
// so this repo defines its own single-file container over the same ncnn content:
//     "FTHRB200" | u64 param_len | param text | bin bytes            (see feathercnn_b200/tools/feathermodel.py)
// InitFromPath(p) accepts that container, or falls back to p + ".param" / p + ".bin".
#pragma once

#include <map>
#include <set>
#include <string>
#include <vector>

#include "layer.h"
#include "ncnn/mat.h"
#include "rt_param.h"

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class Net {
public:
    Net();                             // net.cpp:31-39 of the reference
    explicit Net(size_t num_threads);  // README.md:59 (num_threads is accepted and ignored on the GPU)
    ~Net();

    // ---- reference snapshot API (net.h:33-50) ------------------------------------------------------
    int LoadParam(const char* param_path);
    int LoadParam(FILE* fp);
    int LoadParamFromText(const char* param_text);  // same grammar from memory (README.md:62 "raw buffers")
    int LoadWeights(const char* weights_path);
    int LoadWeights(FILE* fp);
    int FeedInput(const char* input_name, ncnn::Mat& in);  // one image (batch 1), like blob.cpp:70-77
    int Forward();
    // Returns a HOST pointer (a mirror refreshed by this call, valid until the next Extract of that blob).
    int Extract(std::string blob_name, float** output_ptr, int* n, int* c, int* h, int* w);
    int Extract(std::string blob_name, ncnn::Mat& out);  // image 0; copies every channel (the reference's
                                                         // version repeats channel 0, net.cpp:291-294); a Mat of
                                                         // the blob's ncnn rank (Blob::dims)
    int BuildBlobMap();
    std::map<std::string, Blob<float>*> blob_map;

    // ---- README-era API (README.md:56-75) ----------------------------------------------------------
    int InitFromPath(const char* model_path);
    int InitFromFile(FILE* fp);
    int InitFromBuffer(const void* net_buffer, size_t size);
    int InitGraphFromBuffer(const void* net_buffer, size_t size);  // the container's graph only; weights via the arena calls below
    int Forward(const float* input);                 // one image shaped like the model's Input layer
    int Forward(const float* input, int height, int width);
    int ExtractBlob(float* output_ptr, std::string blob_name);
    int GetBlobDataSize(size_t* data_size, std::string blob_name);

    // ---- batched / device API (new) ----------------------------------------------------------------
    int FeedInputBatch(const char* input_name, const float* host_nchw, int n, int c, int h, int w);
    int FeedInputDevice(const char* input_name, const float* device_nchw, int n, int c, int h, int w);
    // u8 images (interleaved, ncnn pixel `type`, mat.h:126-146) -> resize -> planar fp32 -> (x - mean) * norm, on the
    // device, straight into the input blob: ncnn::Mat::from_pixels_resize + substract_mean_normalize + FeedInput for a
    // batch (mat.h:149-160).  mean_vals / norm_vals: host arrays or NULL; target <= 0 keeps w / h.
    int FeedInputPixels(const char* input_name, const unsigned char* host_pixels, int type, int w, int h, int target_w,
                        int target_h, int batch, const float* mean_vals, const float* norm_vals);
    int ForwardBatch(const float* host_nchw, int batch);  // FeedInputBatch(first Input layer) + Forward
    int ExtractDevice(std::string blob_name, const float** device_ptr, int* n, int* c, int* h, int* w);
    int Synchronize();
    // Pipelined end-to-end path (two batches in flight): the H2D copy of a batch runs on a copy stream behind an
    // event while the previous batch computes; Forward follows on the Net's stream, then the D2H copy of `blob_name`
    // (may be NULL) into `host_out`.  `host_nchw` / `host_out` should be pinned and must stay valid until WaitBatch.
    // Returns a ticket (>= 0) for WaitBatch, or a negative error code.
    int SubmitBatch(const float* host_nchw, int batch, const char* blob_name, float* host_out);
    int WaitBatch(int ticket);

    // Weight arena: every weight blob of the model, contiguous on the device.  Rank 0 of a multi-GPU job
    // fills it with LoadWeights(); other ranks call PrepareWeightArena(), receive the bytes (e.g.
    // ncclBroadcast into WeightArena()), then AttachWeights().
    int PrepareWeightArena();
    float* WeightArena() const { return weight_arena_; }
    size_t WeightArenaFloats() const { return weight_arena_floats_; }
    int AttachWeights();

    // Options.
    void SetStream(void* cuda_stream);
    void SetFusion(bool enable) { fusion_ = enable; }  // before LoadParam: conv+ReLU, BN+Scale(+ReLU), eltwise+ReLU
    void SetCudaGraph(bool enable) { use_graph_ = enable; }
    unsigned long long LaunchesPerForward() const { return launches_per_forward_; }
    const std::string& InputName() const { return input_name_; }
    void InputShape(int* c, int* h, int* w) const { *c = input_c_; *h = input_h_; *w = input_w_; }
    std::vector<std::string> BlobNames() const;
    // Runs the SetFusion(true) graph rewrite now instead of at the first Forward (host only, no kernel; idempotent) and
    // returns how many layers were absorbed into their producers.  LayerFusedAway: 1 / 0, -1 for an unknown layer.
    int FuseNow();
    int LayerFusedAway(const std::string& layer_name) const;
    // The FcudaConvAlgo the convolution layer's booster holds (set by Reshape, so valid after a Forward); -1 for an
    // unknown layer, a layer that is not a convolution, or a layer fused away.
    int LayerConvAlgo(const std::string& layer_name) const;

private:
    int ParseParamText(const char* text);
    int LoadWeightsFrom(const ncnn::ModelBin& mb, bool upload);
    int InitLayers();
    int Reshape();
    int RunLayers();
    int BindWeightBlobs(bool upload);
    int ApplyFusion();
    void ResetGraph();
    void FreePipeline();
    struct PipeSlot {
        float* dev = nullptr;
        size_t capacity = 0;
        void *ev_h2d = nullptr, *ev_free = nullptr, *ev_done = nullptr;  // cudaEvent_t
        bool used = false;
    };

    RuntimeParameter<float>* rt_param;
    std::vector<Layer*> layers;
    int _param_loaded;
    int _weights_loaded;
    int _net_initialized;

    float* weight_arena_ = nullptr;
    size_t weight_arena_floats_ = 0;
    std::map<std::string, std::vector<float>> host_mirror_;
    std::string input_name_;
    int input_c_ = 0, input_h_ = 0, input_w_ = 0;
    bool fusion_ = false;
    bool use_graph_ = false;
    std::map<std::vector<size_t>, void*> graph_cache_;  // blob addresses+sizes -> cudaGraphExec_t
    unsigned long long launches_per_forward_ = 0;
    bool owns_stream_ = false;
    bool fusion_applied_ = false;
    std::set<std::vector<size_t>> warmed_keys_;  // graph keys that already ran once eagerly
    float* graph_pool_ptr_ = nullptr;            // scratch pool address the cached graphs were captured with
    int init_precision_ = -1;                    // fcuda precision mode the packed filters were made for
    unsigned char* pixel_stage_ = nullptr;  // device staging of the u8 images of FeedInputPixels
    size_t pixel_stage_bytes_ = 0;
    PipeSlot pipe_[2];
    void* copy_stream_ = nullptr;
    unsigned submitted_ = 0;
};

}  // inline namespace b200
}  // namespace feather
