// InnerProductLayer (mirrors /root/reference/src/layers/inner_product_layer.h:26-171).  The per-image SGEMV
// of the reference becomes one weight-streaming wgmma GEMM over the batch (fcuda_inner_product_forward).
#pragma once

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class InnerProductLayer : public Layer {
public:
    explicit InnerProductLayer(RuntimeParameter<float>* rt_param)
        : Layer(rt_param), weight_data_size(0), input_size(0), output_size(0), bias_term(false), kernel_data(NULL),
          bias_data(NULL), fuse_relu(false), packed(NULL) {
        _fusible = true;
    }
    ~InnerProductLayer() { delete packed; }

    int LoadParam(const ncnn::ParamDict& pd) {
        this->output_size = pd.get(0, 0);
        this->bias_term = pd.get(1, 0);
        this->weight_data_size = pd.get(2, 0);
        if (output_size == 0) return FEATHER_ERR_WEIGHTS;
        this->input_size = this->weight_data_size / this->output_size;
        weights.push_back(NewWeightBlob(this->name + "_weights", output_size, input_size, 1, 1));
        if (this->bias_term) weights.push_back(NewWeightBlob(this->name + "_bias", output_size, 1, 1, 1));
        return 0;
    }

    int LoadWeights(const ncnn::ModelBin& mb) {
        ncnn::Mat weight_data = mb.load(static_cast<int>(weight_data_size), 0);
        if (weight_data.empty() || this->weights.empty()) return FEATHER_ERR_WEIGHTS;
        int rc = this->weights[0]->CopyDataFromMat(weight_data);
        if (rc) return rc;
        if (this->bias_term) {
            ncnn::Mat bias_mat = mb.load(static_cast<int>(output_size), 1);
            if (bias_mat.empty() || this->weights.size() < 2) return FEATHER_ERR_WEIGHTS;
            rc = weights[1]->CopyDataFromMat(bias_mat);
        }
        return rc;
    }

    // ncnn's rule for a rank-2 bottom of w == num_input and h > 1: each row is one input vector (a Transformer's
    // tokens), and the top is rank 2 with w = num_output.  Otherwise each image is one input vector.
    int Reshape() {
        const Blob<float>* bottom_blob = bottoms[0];
        const size_t per_image = bottom_blob->channels() * bottom_blob->height() * bottom_blob->width();
        if (bottom_blob->dims() == 2 && bottom_blob->width() == input_size && bottom_blob->height() > 1) {
            if (bottom_blob->num() * bottom_blob->height() > 0x7fffffffu) return FEATHER_ERR_UNSUPPORTED;
            rows = static_cast<int>(bottom_blob->num() * bottom_blob->height());
            this->tops[0]->ReshapeWithRealloc(static_cast<int>(bottom_blob->num()), 1,
                                              static_cast<int>(bottom_blob->height()), static_cast<int>(output_size));
            this->tops[0]->set_dims(2);
            size_t scratch = 0, dull = 0;
            int rc = fcuda_inner_product_get_buffer_size(static_cast<int>(input_size), static_cast<int>(output_size),
                                                         rows, &scratch, &dull);
            if (rc) return rc;
            MEMPOOL_CHECK_RETURN(this->common_mempool->Request(sizeof(float) * scratch));
            return 0;
        }
        if (input_size != per_image) {
            LOGE("In Layer %s: Bottom %s data size %zu is inconsistant with expected input size %zu.", this->name.c_str(),
                 bottom_blob->name.c_str(), per_image, input_size);
            return FEATHER_ERR_WEIGHTS;
        }
        const int batch = bottom_blob->num();
        rows = batch;
        this->tops[0]->ReshapeWithRealloc(batch, static_cast<int>(output_size), 1, 1);
        size_t scratch = 0, dull = 0;
        int rc = fcuda_inner_product_get_buffer_size(static_cast<int>(input_size), static_cast<int>(output_size), batch,
                                                     &scratch, &dull);
        if (rc) return rc;
        MEMPOOL_CHECK_RETURN(this->common_mempool->Request(sizeof(float) * scratch));
        return 0;
    }

    int Init() {
        size_t scratch = 0, packed_size = 0;
        int rc = fcuda_inner_product_get_buffer_size(static_cast<int>(input_size), static_cast<int>(output_size), 1,
                                                     &scratch, &packed_size);
        if (rc) return rc;
        if (!packed) packed = new Blob<float>(this->name + "_proc_weights");
        packed->ReshapeWithRealloc(1, 1, 1, static_cast<int>(packed_size));
        if (!packed->data() || !weights[0]->data()) return FEATHER_ERR_WEIGHTS;
        rc = fcuda_inner_product_init(static_cast<int>(input_size), static_cast<int>(output_size), packed->data(),
                                      weights[0]->data(), stream());
        if (rc) return rc;
        this->kernel_data = packed->data();
        // the reference dereferences weights[1] even without a bias term (inner_product_layer.h:91)
        this->bias_data = bias_term ? this->weights[1]->data() : NULL;
        return 0;
    }

    int Forward() {
        float* buffer = NULL;
        MEMPOOL_CHECK_RETURN(this->common_mempool->GetPtr(&buffer));
        return fcuda_inner_product_forward(static_cast<int>(input_size), static_cast<int>(output_size), tops[0]->data(),
                                           bottoms[0]->data(), kernel_data, bias_data, buffer, fuse_relu ? 1 : 0, rows,
                                           stream());
    }

    int Fuse(Layer* next_layer) {  // inner_product_layer.h:43-53
        if (next_layer->type.compare("ReLU") == 0) {
            fuse_relu = true;
            return 1;
        }
        return 0;
    }

protected:
    size_t weight_data_size;
    size_t input_size;
    size_t output_size;
    bool bias_term;
    float* kernel_data;
    float* bias_data;
    bool fuse_relu;
    Blob<float>* packed;
    int rows = 0;  // input vectors per Forward: the batch, or batch * h for a rank-2 bottom
};

}  // inline namespace b200
}  // namespace feather
