// Device-resident Blob (see include/feather/blob.h).
#include <feather/blob.h>

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

template <class Dtype>
void Blob<Dtype>::Free() {
    if (_data && _owned) cudaFree(_data);
    _data = nullptr;
    _capacity = 0;
    _owned = true;
}

template <class Dtype>
void Blob<Dtype>::ReshapeWithRealloc(const Blob<Dtype>* p_blob) {
    ReshapeWithRealloc(p_blob->num(), p_blob->channels(), p_blob->height(), p_blob->width());
    _dims = p_blob->dims();
}

template <class Dtype>
void Blob<Dtype>::ReshapeWithRealloc(int num, int channels, int height, int width) {
    const size_t elem_size = static_cast<size_t>(num) * channels * height * width;
    Realloc(elem_size);
    _num = num;
    _channels = channels;
    _height = height;
    _width = width;
    _dims = 3;
}

template <class Dtype>
void Blob<Dtype>::Realloc(size_t elem_size) {
    if (_stage) {  // weight blob: host staging until the Net binds it to the arena
        _host.assign(elem_size, Dtype());
        return;
    }
    if (!_owned) {  // leaving an external view: start owning again
        _data = nullptr;
        _capacity = 0;
        _owned = true;
    }
    if (elem_size > _capacity) {  // grow only, blob.cpp:61-68
        if (_data) cudaFree(_data);
        _data = nullptr;
        void* p = nullptr;
        if (cudaMalloc(&p, (elem_size ? elem_size : 1) * sizeof(Dtype)) != cudaSuccess) {
            LOGE("Blob %s: cudaMalloc of %zu bytes failed", name.c_str(), elem_size * sizeof(Dtype));
            _capacity = 0;
            return;
        }
        _data = static_cast<Dtype*>(p);
        _capacity = elem_size;
    }
}

template <class Dtype>
int Blob<Dtype>::CopyFromMat(const ncnn::Mat& mat) {
    this->ReshapeWithRealloc(1, mat.c, mat.h, mat.w);
    return this->CopyDataFromMat(mat);
}

template <class Dtype>
int Blob<Dtype>::CopyDataFromMat(const ncnn::Mat& mat) {
    if (this->data_size() != static_cast<size_t>(mat.c) * mat.h * mat.w) {
        LOGE("In Blob %s: Mat and target blob shape mismatch. blob shape (%zu %zu %zu %zu), mat shape (%d %d %d)",
             this->name.c_str(), num(), channels(), height(), width(), mat.c, mat.h, mat.w);
        return FEATHER_ERR_BAD_DIMS;
    }
    const size_t plane = static_cast<size_t>(mat.h) * mat.w;
    // repack ncnn's 16-byte aligned channel step into a dense buffer (blob.cpp:86-93)
    std::vector<Dtype> dense;
    const Dtype* src = nullptr;
    if (mat.c <= 1 || mat.cstep == plane) {
        src = static_cast<const Dtype*>(mat.data);
    } else {
        dense.resize(plane * mat.c);
        for (int c = 0; c < mat.c; ++c)
            memcpy(dense.data() + plane * c, static_cast<const unsigned char*>(mat.data) + mat.cstep * c * mat.elemsize,
                   plane * sizeof(Dtype));
        src = dense.data();
    }
    if (_stage) {
        _host.assign(src, src + data_size());
        return 0;
    }
    if (!_data) return FEATHER_ERR_CUDA;
    return cudaMemcpy(_data, src, data_size() * sizeof(Dtype), cudaMemcpyHostToDevice) == cudaSuccess ? 0 : FEATHER_ERR_CUDA;
}

template <class Dtype>
int Blob<Dtype>::CopyFromHost(const Dtype* host, void* stream) {
    if (!_data) return FEATHER_ERR_CUDA;
    cudaError_t e = cudaMemcpyAsync(_data, host, data_size() * sizeof(Dtype), cudaMemcpyHostToDevice,
                                    static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : FEATHER_ERR_CUDA;
}

template <class Dtype>
int Blob<Dtype>::CopyToHost(Dtype* host, void* stream) const {
    if (!_data) return FEATHER_ERR_CUDA;
    cudaError_t e = cudaMemcpyAsync(host, _data, data_size() * sizeof(Dtype), cudaMemcpyDeviceToHost,
                                    static_cast<cudaStream_t>(stream));
    if (e == cudaSuccess) e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? 0 : FEATHER_ERR_CUDA;
}

template <class Dtype>
void Blob<Dtype>::BindExternal(Dtype* device_ptr) {
    if (_data && _owned) cudaFree(_data);
    _data = device_ptr;
    _owned = false;
    _capacity = data_size();
    _stage = false;
    std::vector<Dtype>().swap(_host);
}

template <class Dtype>
void Blob<Dtype>::ViewExternal(Dtype* device_ptr, int num, int channels, int height, int width, int dims) {
    _num = num;
    _dims = dims;
    _channels = channels;
    _height = height;
    _width = width;
    BindExternal(device_ptr);
}

template <class Dtype>
void Blob<Dtype>::PrintBlobInfo() const {
    printf("----BlobShape----\n");
    printf("NCHW=(%zu %zu %zu %zu)\n", _num, _channels, _height, _width);
    printf("----------------\n");
}

template class Blob<float>;
template class Blob<uint16_t>;
template class Blob<char>;

}  // inline namespace b200
}  // namespace feather
