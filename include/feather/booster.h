// booster::ConvBooster — C++ face of the drop-in boundary, same names and call protocol as the reference's
// class (/root/reference/src/booster/include/booster/booster.h:42-170) over the fcuda C ABI.  Differences,
// all forced by batching and the GPU: pointers are device pointers, GetBufferSize/Forward take a batch count,
// Init/Forward take a stream, and sizes are size_t floats.
#pragma once

#include <fcuda.h>
#include <stddef.h>
#include <stdio.h>

namespace booster {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

enum ConvAlgo { NAIVE, IM2COL, SGECONV, DEPTHWISE, WINOGRADF63, WINOGRADF63FUSED, WINOGRADF23 };
enum ActivationType { None, ReLU, Clip };  // Clip == FCUDA_ACT_CLIP: bounds passed to ForwardOpts / ForwardClip

struct ConvParam : FcudaConvParam {
    ConvParam() { *static_cast<FcudaConvParam*>(this) = FcudaConvParam(); }
    void AssignOutputDim() { fcuda_conv_assign_output_dim(this); }   // booster.h:113-125
    void AssignPaddedDim() {                                          // booster.h:126-134
        input_h = input_h + pad_top + pad_bottom;
        input_w = input_w + pad_left + pad_right;
        pad_left = pad_bottom = pad_right = pad_top = 0;
    }
    void LogParams(const char* layer_name) const {                   // booster.h:135-144
        printf("-----Layer %s ConvParam----\n", layer_name);
        printf("Input CxHxW=(%d, %d, %d)\n", input_channels, input_h, input_w);
        printf("Output CxHxW=(%d, %d, %d)\n", output_channels, output_h, output_w);
        printf("Group = %d\n", group);
        printf("Kernel HxW=(%d, %d)\n", kernel_h, kernel_w);
        printf("Stride HxW=(%d, %d)\n", stride_h, stride_w);
        printf("Paddings (%d %d %d %d)\n", pad_left, pad_bottom, pad_right, pad_top);
    }
    double GetFLOPS() const {                                         // booster.h:145-148
        return 2.0 * output_channels * input_channels * output_h * output_w * kernel_h * kernel_w / group;
    }
};

// ConvBooster doesn't allocate any memory (booster.h:155).
class ConvBooster {
public:
    ConvBooster() : algo(-1) {}
    int SelectAlgo(ConvParam* param) { return fcuda_conv_select_algo(param, &algo); }            // reference rule
    int SelectAlgoTuned(ConvParam* param) { return fcuda_conv_select_algo_tuned(param, &algo); }  // tuned cost model
    int ForceSelectAlgo(ConvAlgo a) { algo = static_cast<int>(a); return 0; }
    int SetFuncs() { return algo < 0 ? -1 : 0; }
    int GetBufferSize(ConvParam* param, size_t* buffer_size, size_t* processed_kernel_size, int batch = 1) const {
        return fcuda_conv_get_buffer_size(param, algo, batch, buffer_size, processed_kernel_size);
    }
    int Init(ConvParam* param, float* processed_kernel, const float* kernel, void* stream = nullptr) const {
        return fcuda_conv_init(param, algo, processed_kernel, kernel, stream);
    }
    int Forward(ConvParam* param, float* output, const float* input, const float* kernel, float* buffer,
                const float* bias_arr, int batch = 1, void* stream = nullptr) const {
        return fcuda_conv_forward(param, algo, output, input, kernel, buffer, bias_arr, batch, stream);
    }
    // Forward with everything the epilogue can fuse (fcuda.h, FcudaConvOptions); the two below carry one option each
    int ForwardOpts(ConvParam* param, float* output, const float* input, const float* kernel, float* buffer,
                    const float* bias_arr, const FcudaConvOptions& options, int batch = 1, void* stream = nullptr) const {
        return fcuda_conv_forward_opts(param, algo, output, input, kernel, buffer, bias_arr, &options, batch, stream);
    }
    // Forward + fused Eltwise SUM (+ReLU) of `residual` (same shape as the output)
    int ForwardResidual(ConvParam* param, float* output, const float* input, const float* kernel, float* buffer,
                        const float* bias_arr, const float* residual, int relu_after_add, int batch = 1,
                        void* stream = nullptr) const {
        return fcuda_conv_forward_residual(param, algo, output, input, kernel, buffer, bias_arr, residual, relu_after_add,
                                           batch, stream);
    }
    // Forward with param->activation == Clip: the output clamped to [clip_min, clip_max] in the epilogue
    int ForwardClip(ConvParam* param, float* output, const float* input, const float* kernel, float* buffer,
                    const float* bias_arr, float clip_min, float clip_max, int batch = 1, void* stream = nullptr) const {
        return fcuda_conv_forward_clip(param, algo, output, input, kernel, buffer, bias_arr, clip_min, clip_max, batch,
                                       stream);
    }
    int GetAlgo() const { return algo; }

private:
    int algo;
};

}  // inline namespace b200
}  // namespace booster
