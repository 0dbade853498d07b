/* feather_c.h — C ABI of the host-side feather::Net (libfeather_b200.so) for language bindings.
 * Every function forwards to the C++ method of the same meaning in include/feather/net.h, which in turn mirrors
 * /root/reference/src/net.h:30-70 and README.md:56-75.  Handles are opaque; ints are 0 / negative error codes. */
#ifndef FEATHER_C_H
#define FEATHER_C_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

void* fnet_create(void);                                         /* Net::Net(), net.cpp:31-39 */
void fnet_destroy(void* net);
void fnet_set_fusion(void* net, int enable);                     /* live TryFuse pass, layer.h:61-68 */
void fnet_set_cuda_graph(void* net, int enable);
/* Decodes one ncnn weight blob of `w` floats from an in-memory .bin image (ncnn::ModelBinFromMemory, the loader behind
 * Net::InitFromBuffer; src/ncnn/modelbin.cpp:204-293: type 0 = tagged fp32 / fp16 / 256-entry LUT, type 1 = raw fp32).
 * Host only.  Returns the bytes consumed, or -1 when the blob is rejected (int8, truncated, unknown type). */
long fnet_modelbin_load_mem(const unsigned char* buf, int w, int type, float* out);
int fnet_fuse_now(void* net);                                    /* run the fusion rewrite now; returns #layers absorbed */
int fnet_layer_fused_away(void* net, const char* layer_name);    /* 1 / 0, -1 unknown layer */
/* FcudaConvAlgo a convolution layer runs (after a Forward); -1: unknown layer, not a convolution, or fused away */
int fnet_layer_conv_algo(void* net, const char* layer_name);
void fnet_set_stream(void* net, void* cuda_stream);
int fnet_load_param(void* net, const char* param_path);          /* Net::LoadParam, net.cpp:54-170 */
int fnet_load_param_text(void* net, const char* param_text);     /* same grammar from memory */
int fnet_load_weights(void* net, const char* bin_path);          /* Net::LoadWeights, net.cpp:172-230 */
int fnet_init_from_path(void* net, const char* model_path);      /* README.md:60 */
int fnet_init_from_buffer(void* net, const void* buf, size_t size); /* README.md:62 */
int fnet_prepare_weight_arena(void* net);                        /* non-root ranks: lay out the arena, no file I/O */
int fnet_weight_arena(void* net, float** device_ptr, size_t* floats);
int fnet_attach_weights(void* net);                              /* after the arena was filled (NCCL broadcast) */
int fnet_feed_input_batch(void* net, const char* input_name, const float* host_nchw, int n, int c, int h, int w);
/* u8 images -> (resize) -> planar fp32 -> mean / norm on the device into the input blob (ncnn::Mat::from_pixels_resize +
 * substract_mean_normalize + FeedInput, src/ncnn/mat.h:149-160); mean_vals / norm_vals may be NULL */
int fnet_feed_input_pixels(void* net, const char* input_name, const unsigned char* host_pixels, int type, int w, int h,
                           int target_w, int target_h, int batch, const float* mean_vals, const float* norm_vals);
int fnet_feed_input_device(void* net, const char* input_name, const float* device_nchw, int n, int c, int h, int w);
int fnet_forward(void* net);                                     /* Net::Forward, net.cpp:298-334 */
int fnet_forward_batch(void* net, const float* host_nchw, int batch); /* README.md:65 with a batch */
/* pipelined end-to-end path: H2D on a copy stream behind an event, Forward, D2H of `blob` into host_out; two batches
 * in flight; returns a ticket >= 0 for fnet_wait_batch (Net::SubmitBatch / WaitBatch) */
int fnet_submit_batch(void* net, const float* host_nchw, int batch, const char* blob, float* host_out);
int fnet_wait_batch(void* net, int ticket);
int fnet_synchronize(void* net);
int fnet_blob_shape(void* net, const char* blob, int* n, int* c, int* h, int* w);
/* ncnn rank of one image of the blob (1, 2 or 3); -1 for an unknown blob. */
int fnet_blob_dims(void* net, const char* blob);
int fnet_extract_blob(void* net, const char* blob, float* host_out);  /* README.md:69 */
int fnet_extract_device(void* net, const char* blob, const float** device_ptr, int* n, int* c, int* h, int* w);
unsigned long long fnet_launches_per_forward(void* net);
int fnet_input_shape(void* net, int* c, int* h, int* w);
size_t fnet_blob_names(void* net, char* buf, size_t cap);
const char* fnet_input_name(void* net);


/* ---- feather::NetGroup (include/feather/net_group.h): one model replicated on several GPUs of one box from ONE process:
 * the file is read once, the weight arena reaches the other devices by one ncclBroadcast (dlopen'ed libnccl; peer copies
 * when absent), every batch is sharded contiguously over the devices; no collective in Forward. */
void* fgroup_create(void);
void fgroup_destroy(void* group);
void fgroup_set_options(void* group, int fusion, int cuda_graph);          /* before fgroup_init_from_path */
int fgroup_init_from_path(void* group, const char* model_path, const int* devices, int count); /* NULL / 0: all devices */
int fgroup_size(void* group);
int fgroup_device(void* group, int member);
void* fgroup_member(void* group, int member);                              /* the member's Net handle (fnet_* calls) */
const char* fgroup_broadcast_transport(void* group);                       /* "nccl" | "cudaMemcpyPeer" | "" */
/* shards `batch` host images over the members, gathers `blob` of every image in input order into host_out (may be NULL) */
int fgroup_forward_batch(void* group, const float* host_nchw, int batch, const char* blob, float* host_out);
int fgroup_shard_range(int batch, int members, int member, int* lo, int* hi);  /* rows [lo, hi) of a batch run on `member` */
int fgroup_synchronize(void* group);

#ifdef __cplusplus
}
#endif
#endif
