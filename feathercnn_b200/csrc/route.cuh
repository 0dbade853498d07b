#pragma once
#include <cuda_runtime.h>
namespace fcuda {
constexpr int kRouteMax = 8;

// One channel routing, fcuda_route_forward's FcudaRoute after validation.  Each image of every blob is viewed as
// [outer][extent][inner]; the sources are concatenated along the middle axis (mid = src_begin[num_src] positions),
// shuffled, and positions [first, first + dst_begin[num_dst]) of the shuffled axis go to the destinations in order.
struct RouteGeom {
    const float* src[kRouteMax];
    float* dst[kRouteMax];
    int src_begin[kRouteMax + 1];  // prefix sums of the source extents
    int dst_begin[kRouteMax + 1];  // prefix sums of the destination extents
    int num_src, num_dst;
    int first;                     // first shuffled position the destinations take
    int g, cpg;                    // shuffled position p reads concatenated position (p % g) * cpg + p / g
    int outer, inner;              // inner in floats
};
int route_forward(const RouteGeom& g, int batch, cudaStream_t s);
}  // namespace fcuda
