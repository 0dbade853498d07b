// ShuffleChannelLayer and SliceLayer — ncnn's layers of those names, which ShuffleNet v1 / v2 need; the reference has
// neither.  Both run on fcuda_route_forward, and so does the chain Net::ApplyFusion builds from them: the last layer of
// Concat (axis 0) -> ShuffleChannel -> Slice (axis 0), or of any two adjacent of them, takes the Concat's bottoms and
// the ShuffleChannel's group and writes its own tops from them in one launch.
//
// ShuffleChannel: 0=group (default 1), 1=reverse (default 0); rank-3 bottoms only.  With k = reverse ? C / group : group
// and cpg = C / k, top channel k * j + i is bottom channel cpg * i + j.  C % group != 0 fails at Reshape; k == 1 makes
// the top a view of the bottom.
// Slice: -23300=slices (one entry per top), 1=axis (default 0, ncnn's per-rank axis; fcuda_slice_plan states the rule).
// ncnn's newer 2=indices form is rejected.  Each top keeps the bottom's rank.
#pragma once

#include <vector>

#include <fcuda.h>
#include <feather/layer.h>

namespace feather {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

class RouteLayer : public Layer {
public:
    explicit RouteLayer(RuntimeParameter<float>* rt_param) : Layer(rt_param) {}
    bool absorbed() const { return absorbed_; }
    bool shuffles() const { return shuffle_; }
    // Net::ApplyFusion: this layer's bottom was the top of a Concat on axis 0 with these bottoms, or of a ShuffleChannel
    // (itself perhaps fused with such a Concat); the producer's bottoms and group become this layer's.
    void Absorb(const std::vector<Blob<float>*>& sources, bool shuffle, int group, int reverse) {
        bottoms = sources;
        if (shuffle) {
            shuffle_ = true;
            group_ = group;
            reverse_ = reverse;
        }
        absorbed_ = true;
    }
    int group() const { return group_; }
    int reverse() const { return reverse_; }

protected:
    // The bottoms as one blob concatenated along per-rank `axis`: the same rank and images, equal extents off the axis
    // (Concat's checks).  Gives the rank, the storage axis and the concatenated (c, h, w).
    int View(int axis, int* rank, int* storage_axis, int dims[3]) const {
        const Blob<float>* b0 = bottoms[0];
        *rank = b0->dims();
        const int a = axis < 0 ? axis + *rank : axis;
        if (a < 0 || a >= *rank) {
            LOGE("%s layer %s: axis %d is out of range for rank %d", type.c_str(), name.c_str(), axis, *rank);
            return FEATHER_ERR_UNSUPPORTED;
        }
        const int sa = a + 3 - *rank;
        *storage_axis = sa;
        dims[0] = static_cast<int>(b0->channels());
        dims[1] = static_cast<int>(b0->height());
        dims[2] = static_cast<int>(b0->width());
        for (size_t i = 1; i < bottoms.size(); ++i) {
            const Blob<float>* b = bottoms[i];
            const int d[3] = {static_cast<int>(b->channels()), static_cast<int>(b->height()), static_cast<int>(b->width())};
            bool ok = b->dims() == *rank && b->num() == b0->num();
            for (int k = 0; k < 3; ++k) ok = ok && (k == sa || d[k] == dims[k]);
            if (!ok) {
                LOGE("%s layer %s: concatenated bottoms of different shapes", type.c_str(), name.c_str());
                return FEATHER_ERR_WEIGHTS;
            }
            dims[sa] += d[sa];
        }
        if (shuffle_ && (*rank != 3 || sa != 0 || dims[0] % group_ != 0)) {
            LOGE("%s layer %s: ShuffleChannel group %d needs a rank-3 blob whose %d channels it divides", type.c_str(),
                 name.c_str(), group_, dims[0]);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    // Tops [t0, t0 + 8) per launch; `sizes` are the tops' extents along storage axis `sa` of the view `dims`.
    int Route(int sa, const int dims[3], const std::vector<int>& sizes) {
        FcudaRoute r = {};
        r.outer = 1;
        r.inner = 1;
        for (int k = 0; k < sa; ++k) r.outer *= dims[k];
        for (int k = sa + 1; k < 3; ++k) r.inner *= dims[k];
        r.num_src = static_cast<int>(bottoms.size());
        for (int k = 0; k < r.num_src && k < FCUDA_ROUTE_MAX; ++k) {
            const Blob<float>* b = bottoms[k];
            const size_t d[3] = {b->channels(), b->height(), b->width()};
            r.src[k] = b->data();
            r.src_extent[k] = static_cast<int>(d[sa]);
        }
        r.group = shuffle_ ? group_ : 1;
        r.reverse = shuffle_ ? reverse_ : 0;
        int begin = 0;
        for (size_t t0 = 0; t0 < tops.size(); t0 += FCUDA_ROUTE_MAX) {
            r.dst_begin = begin;
            r.num_dst = 0;
            for (size_t t = t0; t < tops.size() && t < t0 + FCUDA_ROUTE_MAX; ++t, ++r.num_dst) {
                r.dst[r.num_dst] = tops[t]->data();
                r.dst_extent[r.num_dst] = sizes[t];
                begin += sizes[t];
            }
            const int rc = fcuda_route_forward(&r, static_cast<int>(bottoms[0]->num()), stream());
            if (rc) return rc;
        }
        return 0;
    }

    bool absorbed_ = false;
    bool shuffle_ = false;
    int group_ = 1, reverse_ = 0;
};

class ShuffleChannelLayer : public RouteLayer {
public:
    explicit ShuffleChannelLayer(RuntimeParameter<float>* rt_param) : RouteLayer(rt_param) { shuffle_ = true; }
    int LoadParam(const ncnn::ParamDict& pd) {
        group_ = pd.get(0, 1);
        reverse_ = pd.get(1, 0);
        if (group_ < 1) {
            LOGE("ShuffleChannel layer %s: group %d < 1", name.c_str(), group_);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int Reshape() {
        int rank = 0, sa = 0, dims[3];
        const int rc = View(0, &rank, &sa, dims);
        if (rc) return rc;
        const Blob<float>* b = bottoms[0];
        view_ = bottoms.size() == 1 && (reverse_ ? dims[0] / group_ : group_) == 1;
        if (view_) {
            tops[0]->ViewExternal(b->data(), b->num(), b->channels(), b->height(), b->width(), 3);
            return 0;
        }
        tops[0]->ReshapeWithRealloc(b->num(), dims[0], dims[1], dims[2]);
        tops[0]->set_dims(3);
        sizes_.assign(1, dims[0]);
        dims_[0] = dims[0]; dims_[1] = dims[1]; dims_[2] = dims[2];
        return 0;
    }
    int Forward() { return view_ ? 0 : Route(0, dims_, sizes_); }

private:
    bool view_ = false;
    int dims_[3] = {0, 0, 0};
    std::vector<int> sizes_;
};

class SliceLayer : public RouteLayer {
public:
    explicit SliceLayer(RuntimeParameter<float>* rt_param) : RouteLayer(rt_param) {}
    int LoadParam(const ncnn::ParamDict& pd) {
        if (pd.has(2)) {
            LOGE("Slice layer %s: 2=indices is not supported; give the sizes as -23300=", name.c_str());
            return FEATHER_ERR_UNSUPPORTED;
        }
        const ncnn::Mat s = pd.get(0, ncnn::Mat());
        const int n = s.empty() ? 0 : s.w;
        if (tops.empty() || n != static_cast<int>(tops.size())) {
            LOGE("Slice layer %s: %d slices for %zu tops", name.c_str(), n, tops.size());
            return FEATHER_ERR_UNSUPPORTED;
        }
        slices_.assign(static_cast<const int*>(s.data), static_cast<const int*>(s.data) + n);
        for (int v : slices_)
            if (v != -233 && v < 1) {
                LOGE("Slice layer %s: slice size %d (sizes are >= 1, or -233 for an even share)", name.c_str(), v);
                return FEATHER_ERR_UNSUPPORTED;
            }
        axis_ = pd.get(1, 0);
        if (axis_ < -3 || axis_ > 2) {
            LOGE("Slice layer %s: axis %d is out of range", name.c_str(), axis_);
            return FEATHER_ERR_UNSUPPORTED;
        }
        return 0;
    }
    int axis() const { return axis_; }
    int Reshape() {
        int rank = 0, sa = 0;
        int rc = View(axis_, &rank, &sa, dims_);
        if (rc) return rc;
        sizes_.resize(slices_.size());
        rc = fcuda_slice_plan(rank, axis_, dims_, slices_.data(), static_cast<int>(slices_.size()), &sa_, sizes_.data());
        if (rc) {
            LOGE("Slice layer %s: the slices do not fit the %d positions of axis %d", name.c_str(), dims_[sa], axis_);
            return rc;
        }
        for (size_t t = 0; t < tops.size(); ++t) {
            int d[3] = {dims_[0], dims_[1], dims_[2]};
            d[sa_] = sizes_[t];
            tops[t]->ReshapeWithRealloc(bottoms[0]->num(), d[0], d[1], d[2]);
            tops[t]->set_dims(rank);
        }
        return 0;
    }
    int Forward() { return Route(sa_, dims_, sizes_); }

private:
    std::vector<int> slices_;
    int axis_ = 0;
    int sa_ = 0;
    int dims_[3] = {0, 0, 0};
    std::vector<int> sizes_;
};

}  // inline namespace b200
}  // namespace feather
