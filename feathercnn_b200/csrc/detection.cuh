#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "fcuda.h"

namespace fcuda {
// ncnn Permute of `batch` (c, h, w) images; order_type 0-5 as in include/fcuda.h.  Order 3 is a tiled transpose.
int permute_forward(const float* in, float* out, int c, int h, int w, int order, int batch, cudaStream_t s);
// Max-subtracted softmax over the middle axis of `batch` (outer, len, inner) views.
int softmax_axis_forward(const float* in, float* out, int outer, int len, int inner, int batch, cudaStream_t s);
// Caffe / ncnn PriorBox of a feat_w x feat_h map: out is (2, 4 * priors) floats, boxes then variances.
int priorbox_forward(float* out, const FcudaPriorBoxParam& p, int per_loc, int feat_w, int feat_h, float img_w, float img_h,
                     float step_w, float step_h, cudaStream_t s);
// Centre-size decode of `batch` images of `num_priors` loc rows against one priors blob.
int ssd_decode(float* boxes, const float* loc, const float* priors, int num_priors, int batch, cudaStream_t s);
// Workspace (floats) of detection_output.
size_t detection_output_workspace(int num_priors, int num_classes, int nms_top_k, int batch);
int detection_output(float* out, const float* loc, const float* conf, const float* priors, int num_priors, int num_classes,
                     float conf_threshold, float nms_threshold, int nms_top_k, int keep_top_k, float* workspace, int batch,
                     cudaStream_t s);
// YOLO head (include/fcuda.h, FcudaYoloParam); the parameters are checked by the caller.
int yolo_decode(float* scores, int* classes, float* boxes, const float* const* inputs, const FcudaYoloParam& p, int batch,
                cudaStream_t s);
// Workspace (floats) of yolo_detection.
size_t yolo_detection_workspace(int slots, int batch);
// decode, select, suppression mask, sweep: four launches.
int yolo_detection(float* out, const float* const* inputs, const FcudaYoloParam& p, float* workspace, int batch,
                   cudaStream_t s);
// Faster R-CNN (include/fcuda.h, FcudaProposalParam); the parameters are checked by the caller.  The 9 anchors of p as
// (x1, y1, w, h) rows, host only.
void proposal_anchors(const FcudaProposalParam& p, float* table);
int proposal_decode(float* boxes, const float* score, const float* bbox, const float* im_info, const FcudaProposalParam& p,
                    int feat_h, int feat_w, int batch, cudaStream_t s);
// Workspace (floats) of proposal_forward.
size_t proposal_workspace(const FcudaProposalParam& p, int feat_h, int feat_w, int batch);
// decode, select, suppression mask, sweep: four launches.
int proposal_forward(float* rois, float* scores, const float* score, const float* bbox, const float* im_info,
                     const FcudaProposalParam& p, int feat_h, int feat_w, float* workspace, int batch, cudaStream_t s);
int roi_pooling_forward(float* out, const float* in, const float* rois, int channels, int height, int width, int num_rois,
                        int pooled_h, int pooled_w, float spatial_scale, int batch, cudaStream_t s);
// R-FCN; channels == output_dim * pooled_h * pooled_w, checked by the caller.
int psroi_pooling_forward(float* out, const float* in, const float* rois, int channels, int height, int width,
                          int num_rois, int pooled_h, int pooled_w, int output_dim, float spatial_scale, int batch,
                          cudaStream_t s);
}  // namespace fcuda
