// ncnn::ParamDict — the per-layer "id=value" dictionary of the ncnn .param format
// (/root/reference/src/ncnn/paramdict.h, paramdict.cpp:34-174).  Re-implemented; same get/set surface.
#pragma once

#include <stdio.h>

#include "mat.h"

namespace ncnn {
inline namespace b200 {  // ABI tag: keeps these symbols apart from the reference build when both are loaded

// ncnn's own limit; Deconvolution's output_w / output_h are ids 20 / 21
#define NCNN_MAX_PARAM_COUNT 32

class ParamDict {
public:
    ParamDict() { clear(); }
    bool has(int id) const { return params[id].loaded != 0; }  // the id appeared on the layer's line
    int get(int id, int def) const { return params[id].loaded ? params[id].i : def; }
    float get(int id, float def) const { return params[id].loaded ? params[id].f : def; }
    Mat get(int id, const Mat& def) const { return params[id].loaded ? params[id].v : def; }
    void set(int id, int i) { params[id].loaded = 1; params[id].i = i; }
    void set(int id, float f) { params[id].loaded = 1; params[id].f = f; }
    void set(int id, const Mat& v) { params[id].loaded = 1; params[id].v = v; }
    void clear();
    // Parses "id=value" pairs up to the end of the current line (text .param), paramdict.cpp:92-174.
    int load_param(FILE* fp);
    // Same from a memory cursor (advanced past the consumed text), paramdict.cpp:198+.
    int load_param_mem(const char*& mem);

private:
    struct Entry {
        int loaded;
        union { int i; float f; };
        Mat v;
    } params[NCNN_MAX_PARAM_COUNT];
};

}  // inline namespace b200
}  // namespace ncnn
