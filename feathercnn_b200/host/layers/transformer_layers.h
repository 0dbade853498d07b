// LayerNormLayer, MemoryDataLayer and MultiHeadAttentionLayer: ncnn's layers of those names, what a Vision Transformer
// exported by pnnx needs beyond the convolution engine (the reference has none of them).  Token blobs are rank 2: w =
// features, h = tokens.  Parameter ids and defaults follow ncnn's operator table.  None of them takes part in fusion.
#pragma once

#include <cuda_runtime.h>
#include <fcuda.h>
#include <feather/layer.h>

#include <math.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// 0 = affine_size, 1 = eps (0.001), 2 = affine (1).  Weights: gamma, beta (affine_size raw floats each).
class LayerNormLayer : public Layer {
public:
    explicit LayerNormLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        affine_size = pd.get(0, 0);
        eps = pd.get(1, 0.001f);
        affine = pd.get(2, 1);
        if (affine_size < 1 || !(eps >= 0.f) || !isfinite(eps) || (affine != 0 && affine != 1) || bottoms.size() != 1 ||
            tops.size() != 1) {
            LOGE("LayerNorm layer %s: affine_size %d, eps %g, affine %d with %zu bottoms and %zu tops is not supported",
                 this->name.c_str(), affine_size, eps, affine, bottoms.size(), tops.size());
            return FEATHER_ERR_UNSUPPORTED;
        }
        if (affine) {
            weights.push_back(NewWeightBlob(this->name + "_gamma", 1, 1, 1, affine_size));
            weights.push_back(NewWeightBlob(this->name + "_beta", 1, 1, 1, affine_size));
        }
        return 0;
    }
    int LoadWeights(const ncnn::ModelBin& mb) {
        if (!affine) return 0;
        ncnn::Mat gamma = mb.load(affine_size, 1);
        ncnn::Mat beta = mb.load(affine_size, 1);
        if (gamma.empty() || beta.empty()) return FEATHER_ERR_WEIGHTS;
        const int rc = weights[0]->CopyDataFromMat(gamma);
        return rc ? rc : weights[1]->CopyDataFromMat(beta);
    }
    // Rank 2: each row (affine_size == w).  Rank 3: each row (affine_size == w) or each channel plane (== w * h).
    int Reshape() {
        const Blob<float>* b = bottoms[0];
        const size_t w = b->width(), plane = b->width() * b->height();
        const size_t n = static_cast<size_t>(affine_size);
        if ((b->dims() != 2 && b->dims() != 3) || (n != w && (b->dims() != 3 || n != plane))) {
            LOGE("LayerNorm layer %s: affine_size %d does not match a rank-%d blob of w %zu, h %zu", this->name.c_str(),
                 affine_size, b->dims(), b->width(), b->height());
            return FEATHER_ERR_UNSUPPORTED;
        }
        tops[0]->ReshapeWithRealloc(b);
        return 0;
    }
    int Forward() {
        const Blob<float>* b = bottoms[0];
        return fcuda_layer_norm_forward(tops[0]->data(), b->data(), affine_size,
                                        static_cast<long long>(b->data_size() / affine_size),
                                        affine ? weights[0]->data() : NULL, affine ? weights[1]->data() : NULL, eps,
                                        stream());
    }

private:
    int affine_size = 0, affine = 1;
    float eps = 0.001f;
};

// 0 = w, 1 = h, 2 = c: the rank is the number of leading dims given (c gives rank 3, h rank 2, w rank 1).  Data: w * h
// * c raw floats.  The top holds one copy per image of the net's current batch (Net::Reshape passes it in), so
// BinaryOp / Concat see operands of equal batch.  The copies are written on the device when the batch or the top's
// storage changes; Reshape runs before every Forward and outside any graph capture, so a replayed graph reads them.
class MemoryDataLayer : public Layer {
public:
    explicit MemoryDataLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        w = pd.get(0, 0);
        h = pd.get(1, 0);
        c = pd.get(2, 0);
        const int d = pd.get(11, 0);
        rank = c ? 3 : h ? 2 : w ? 1 : 0;
        if (d != 0 || rank == 0 || w < 1 || (rank >= 2 && h < 1) || c < 0 || !bottoms.empty() || tops.size() != 1) {
            LOGE("MemoryData layer %s: w %d, h %d, c %d, d %d with %zu bottoms and %zu tops is not supported (w, h, c "
                 "positive, no depth; no bottom, one top)", this->name.c_str(), w, h, c, d, bottoms.size(), tops.size());
            return FEATHER_ERR_UNSUPPORTED;
        }
        weights.push_back(NewWeightBlob(this->name + "_data", 1, dim_c(), dim_h(), w));
        return 0;
    }
    int LoadWeights(const ncnn::ModelBin& mb) {
        ncnn::Mat data = mb.load(w * dim_h() * dim_c(), 1);
        if (data.empty()) return FEATHER_ERR_WEIGHTS;
        return weights[0]->CopyDataFromMat(data);
    }
    void set_batch(int n) { batch = n > 0 ? n : 1; }
    int Reshape() {
        Blob<float>* t = tops[0];
        t->ReshapeWithRealloc(batch, dim_c(), dim_h(), w);
        t->set_dims(rank);
        if (!t->data() || !weights[0]->data()) return FEATHER_ERR_WEIGHTS;
        if (t->data() == filled_ptr && batch == filled_batch) return 0;
        // copy 1, then double the filled prefix: ceil(log2(batch)) + 1 device-to-device copies
        const size_t one = weights[0]->data_size() * sizeof(float);
        cudaStream_t s = static_cast<cudaStream_t>(stream());
        char* dst = reinterpret_cast<char*>(t->data());
        if (cudaMemcpyAsync(dst, weights[0]->data(), one, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
            return FEATHER_ERR_CUDA;
        for (size_t have = 1; have < static_cast<size_t>(batch); have *= 2) {
            const size_t copy = have < batch - have ? have : batch - have;
            if (cudaMemcpyAsync(dst + have * one, dst, copy * one, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
                return FEATHER_ERR_CUDA;
        }
        filled_ptr = t->data();
        filled_batch = batch;
        return 0;
    }
    int Forward() { return 0; }

private:
    int dim_h() const { return rank >= 2 ? h : 1; }
    int dim_c() const { return rank == 3 ? c : 1; }
    int w = 0, h = 0, c = 0, rank = 0;
    int batch = 1;
    const float* filled_ptr = NULL;
    int filled_batch = 0;
};

// 0 = embed_dim, 1 = num_heads, 2 = weight_data_size (embed_dim^2), 3 = kdim, 4 = vdim (embed_dim), 5 = attn_mask (0
// only), 6 = scale (1 / sqrt(head_dim)).  Weights: q_w [E][E], q_b, k_w [E][kdim], k_b, v_w [E][vdim], v_b, out_w
// [E][E], out_b; each matrix flagged, each bias raw.  One bottom (q = k = v) or three (q, k, v), rank 2 (w = features,
// h = sequence).  With one bottom the three input projections are one InnerProduct GEMM over [Wq; Wk; Wv] writing
// [N L][3E], which fcuda_attention_forward reads in place (ld = 3E).
class MultiHeadAttentionLayer : public Layer {
public:
    explicit MultiHeadAttentionLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    ~MultiHeadAttentionLayer() {
        for (Blob<float>* b : packed) delete b;
        delete qkv_raw;
    }
    int LoadParam(const ncnn::ParamDict& pd) {
        embed = pd.get(0, 0);
        heads = pd.get(1, 1);
        const int wds = pd.get(2, 0);
        kdim = pd.get(3, embed);
        vdim = pd.get(4, embed);
        const int mask = pd.get(5, 0);
        const int hd = heads > 0 && embed % heads == 0 ? embed / heads : 0;
        scale = pd.get(6, hd > 0 ? 1.f / sqrtf(static_cast<float>(hd)) : 1.f);
        const bool one = bottoms.size() == 1;
        if (embed < 1 || heads < 1 || hd == 0 || hd % 16 != 0 || hd > 128 || static_cast<long long>(wds) !=
            static_cast<long long>(embed) * embed || kdim < 1 || vdim < 1 || mask != 0 || (!one && bottoms.size() != 3) ||
            (one && (kdim != embed || vdim != embed)) || tops.size() != 1 || scale == 0.f || !isfinite(scale)) {
            LOGE("MultiHeadAttention layer %s: embed_dim %d, num_heads %d, weight_data_size %d, kdim %d, vdim %d, "
                 "attn_mask %d, scale %g with %zu bottoms is not supported (head_dim a multiple of 16 up to 128, "
                 "weight_data_size embed_dim^2, no mask, one or three bottoms)", this->name.c_str(), embed, heads, wds,
                 kdim, vdim, mask, scale, bottoms.size());
            return FEATHER_ERR_UNSUPPORTED;
        }
        const int in[4] = {embed, kdim, vdim, embed};
        const char* tag[4] = {"_q", "_k", "_v", "_out"};
        for (int i = 0; i < 4; ++i) {
            weights.push_back(NewWeightBlob(this->name + tag[i] + "_weight", embed, in[i], 1, 1));
            weights.push_back(NewWeightBlob(this->name + tag[i] + "_bias", embed, 1, 1, 1));
        }
        return 0;
    }
    int LoadWeights(const ncnn::ModelBin& mb) {
        const int in[4] = {embed, kdim, vdim, embed};
        for (int i = 0; i < 4; ++i) {
            ncnn::Mat wm = mb.load(embed * in[i], 0);
            ncnn::Mat bm = mb.load(embed, 1);
            if (wm.empty() || bm.empty()) return FEATHER_ERR_WEIGHTS;
            int rc = weights[2 * i]->CopyDataFromMat(wm);
            if (!rc) rc = weights[2 * i + 1]->CopyDataFromMat(bm);
            if (rc) return rc;
        }
        return 0;
    }
    int Reshape() {
        const Blob<float>* q = bottoms[0];
        const Blob<float>* k = bottoms[fused() ? 0 : 1];
        const Blob<float>* v = bottoms[fused() ? 0 : 2];
        if (q->dims() != 2 || k->dims() != 2 || v->dims() != 2 || q->width() != static_cast<size_t>(embed) ||
            k->width() != static_cast<size_t>(kdim) || v->width() != static_cast<size_t>(vdim) ||
            k->height() != v->height() || k->num() != q->num() || v->num() != q->num() ||
            static_cast<long long>(heads) * ((q->height() + 63) / 64) > 65535 ||
            q->num() * (q->height() > k->height() ? q->height() : k->height()) > 0x7fffffffu) {
            LOGE("MultiHeadAttention layer %s: bottoms do not match embed_dim %d, kdim %d, vdim %d (rank 2, equal "
                 "batch, k and v of one length)", this->name.c_str(), embed, kdim, vdim);
            return FEATHER_ERR_UNSUPPORTED;
        }
        n = static_cast<int>(q->num());
        lq = static_cast<int>(q->height());
        lk = static_cast<int>(k->height());
        tops[0]->ReshapeWithRealloc(n, 1, lq, embed);
        tops[0]->set_dims(2);
        // scratch: [projections | attention output | InnerProduct scratch], each 256-byte aligned
        const size_t rq = static_cast<size_t>(n) * lq, rk = static_cast<size_t>(n) * lk;
        proj_floats = fused() ? align(rq * 3 * embed) : align(rq * embed) + 2 * align(rk * embed);
        attn_floats = align(rq * embed);
        size_t need = 0;
        const int ins[4] = {embed, kdim, vdim, embed};
        const int outs[4] = {fused() ? 3 * embed : embed, embed, embed, embed};
        const size_t rows[4] = {rq, rk, rk, rq};
        for (int i = 0; i < 4; ++i) {
            if (fused() && (i == 1 || i == 2)) continue;
            size_t scratch = 0;
            const int rc = fcuda_inner_product_get_buffer_size(ins[i], outs[i], static_cast<int>(rows[i]), &scratch, NULL);
            if (rc) return rc;
            if (scratch > need) need = scratch;
        }
        MEMPOOL_CHECK_RETURN(this->common_mempool->Request(sizeof(float) * (proj_floats + attn_floats + need)));
        return 0;
    }
    int Init() {
        const int ins[4] = {embed, kdim, vdim, embed};
        cudaStream_t s = static_cast<cudaStream_t>(stream());
        if (fused()) {  // [Wq; Wk; Wv] and [bq; bk; bv] side by side for one projection GEMM
            const size_t ee = static_cast<size_t>(embed) * embed;
            if (!qkv_raw) qkv_raw = new Blob<float>(this->name + "_qkv");
            qkv_raw->ReshapeWithRealloc(1, 1, 1, static_cast<int>(3 * ee + 3 * embed));
            float* dst = qkv_raw->data();
            if (!dst) return FEATHER_ERR_WEIGHTS;
            for (int i = 0; i < 3; ++i) {
                if (cudaMemcpyAsync(dst + i * ee, weights[2 * i]->data(), ee * sizeof(float), cudaMemcpyDeviceToDevice,
                                    s) != cudaSuccess ||
                    cudaMemcpyAsync(dst + 3 * ee + i * embed, weights[2 * i + 1]->data(), embed * sizeof(float),
                                    cudaMemcpyDeviceToDevice, s) != cudaSuccess)
                    return FEATHER_ERR_CUDA;
            }
        }
        for (int i = 0; i < 4; ++i) {
            if (fused() && (i == 1 || i == 2)) continue;
            const int in = ins[i], out = fused() && i == 0 ? 3 * embed : embed;
            size_t packed_size = 0;
            int rc = fcuda_inner_product_get_buffer_size(in, out, 1, NULL, &packed_size);
            if (rc) return rc;
            if (!packed[i]) packed[i] = new Blob<float>(this->name + "_packed");
            packed[i]->ReshapeWithRealloc(1, 1, 1, static_cast<int>(packed_size));
            const float* raw = fused() && i == 0 ? qkv_raw->data() : weights[2 * i]->data();
            if (!packed[i]->data() || !raw) return FEATHER_ERR_WEIGHTS;
            rc = fcuda_inner_product_init(in, out, packed[i]->data(), raw, s);
            if (rc) return rc;
        }
        return 0;
    }
    int Forward() {
        float* pool = NULL;
        MEMPOOL_CHECK_RETURN(this->common_mempool->GetPtr(&pool));
        float* proj = pool;
        float* attn = pool + proj_floats;
        float* scratch = attn + attn_floats;
        const int rq = n * lq, rk = n * lk;
        void* s = stream();
        int rc;
        if (fused()) {
            const float* bias = qkv_raw->data() + 3 * static_cast<size_t>(embed) * embed;
            rc = fcuda_inner_product_forward(embed, 3 * embed, proj, bottoms[0]->data(), packed[0]->data(), bias, scratch,
                                             0, rq, s);
            if (!rc)
                rc = fcuda_attention_forward(attn, proj, 3 * embed, proj + embed, 3 * embed, proj + 2 * embed, 3 * embed,
                                             n, heads, embed / heads, lq, lk, scale, s);
        } else {
            float* qp = proj;
            float* kp = qp + align(static_cast<size_t>(rq) * embed);
            float* vp = kp + align(static_cast<size_t>(rk) * embed);
            float* dst[3] = {qp, kp, vp};
            const int ins[3] = {embed, kdim, vdim};
            const int rows[3] = {rq, rk, rk};
            rc = 0;
            for (int i = 0; i < 3 && !rc; ++i)
                rc = fcuda_inner_product_forward(ins[i], embed, dst[i], bottoms[i]->data(), packed[i]->data(),
                                                 weights[2 * i + 1]->data(), scratch, 0, rows[i], s);
            if (!rc)
                rc = fcuda_attention_forward(attn, qp, embed, kp, embed, vp, embed, n, heads, embed / heads, lq, lk, scale,
                                             s);
        }
        if (rc) return rc;
        return fcuda_inner_product_forward(embed, embed, tops[0]->data(), attn, packed[3]->data(), weights[7]->data(),
                                           scratch, 0, rq, s);
    }

private:
    bool fused() const { return bottoms.size() == 1; }
    static size_t align(size_t floats) { return (floats + 63) / 64 * 64; }
    int embed = 0, heads = 1, kdim = 0, vdim = 0;
    float scale = 1.f;
    int n = 0, lq = 0, lk = 0;
    size_t proj_floats = 0, attn_floats = 0;
    Blob<float>* packed[4] = {NULL, NULL, NULL, NULL};
    Blob<float>* qkv_raw = NULL;
};

}  // inline namespace b200
}  // namespace feather
