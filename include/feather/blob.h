// feather::Blob<Dtype> — owning NCHW tensor (mirrors /root/reference/src/blob.h:26-121), DEVICE resident.
//   * data() is a device pointer (cudaMalloc, 256-byte aligned; the reference used 32-byte host memory).
//   * grow-only reallocation like Blob::Realloc (blob.cpp:61-68).
//   * num() is a real batch dimension (the reference forces 1, blob.cpp:73).
//   * weight blobs first live in a host staging vector (CopyDataFromMat) and are bound to a slice of the
//     Net's device weight arena by Net::LoadWeights (one upload / one NCCL broadcast for the whole model).
#pragma once

#include <stddef.h>

#include <string>
#include <vector>

#include "ncnn/mat.h"
#include "utils.h"

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

template <class Dtype>
class Blob {
public:
    Blob() : name(), _data(nullptr), _capacity(0), _owned(true), _num(0), _channels(0), _height(0), _width(0), _dims(3) {}
    explicit Blob(std::string name)
        : name(name), _data(nullptr), _capacity(0), _owned(true), _num(0), _channels(0), _height(0), _width(0), _dims(3) {}
    ~Blob() { Free(); }
    Blob(const Blob&) = delete;
    Blob& operator=(const Blob&) = delete;

    void Free();
    // Copies p_blob's shape and rank.
    void ReshapeWithRealloc(const Blob<Dtype>* p_blob);
    // Rank 3 (every layer that computes its own (c, h, w) top).
    void ReshapeWithRealloc(int num, int channels, int height, int width);
    void Realloc(size_t elem_size);

    // Host Mat -> device blob of shape (1, c, h, w) (blob.cpp:70-77).
    int CopyFromMat(const ncnn::Mat& src_mat);
    // Host Mat -> this blob's storage (shape must already match, blob.cpp:79-95).  For weight blobs (see
    // StageOnHost) the data is kept on the host until the Net binds it to the device arena.
    int CopyDataFromMat(const ncnn::Mat& src_mat);
    // Dense host buffer (n*c*h*w elements) <-> device.
    int CopyFromHost(const Dtype* host, void* stream = nullptr);
    int CopyToHost(Dtype* host, void* stream = nullptr) const;

    // Weight staging / arena binding.
    void StageOnHost(bool enable) { _stage = enable; }
    bool staged() const { return !_host.empty(); }
    const std::vector<Dtype>& host_stage() const { return _host; }
    void BindExternal(Dtype* device_ptr);  // non-owning; drops the host stage
    // Non-owning view of caller-provided device memory with the given shape (Net::FeedInputDevice).
    void ViewExternal(Dtype* device_ptr, int num, int channels, int height, int width, int dims = 3);
    // ncnn rank of one image: 1 = Mat(w), stored as (c=1, h=1, w); 2 = Mat(w, h), stored as (c=1, h, w); 3 = Mat(w, h, c).
    // Storage does not depend on it; it gives ncnn's per-rank axis numbers (Concat, Softmax) and Extract's Mat their
    // meaning.
    int dims() const { return _dims; }
    void set_dims(int dims) { _dims = dims; }

    Dtype* data() const { return _data; }
    size_t data_size() const { return _num * _channels * _height * _width; }
    size_t num() const { return _num; }
    size_t channels() const { return _channels; }
    size_t height() const { return _height; }
    size_t width() const { return _width; }
    void PrintBlobInfo() const;

    std::string name;

private:
    Dtype* _data;
    size_t _capacity;  // elements
    bool _owned;
    bool _stage = false;
    std::vector<Dtype> _host;
    size_t _num, _channels, _height, _width;
    int _dims;
};

}  // inline namespace b200
}  // namespace feather
