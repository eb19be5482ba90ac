// Exact fixed-point triangle coverage shared by normal_render.cu and dataset_render.cu (the rules are written in
// normal_render.cu's header; dataset_render.cu's header generalises them to S samples per pixel).
//
// A vertex record is int4 (X, Y, z_w bits, ok): window position snapped to 1/256 pixel, window depth z_w in [0, 1]
// for the depth test, ok = 0 when the vertex cannot be drawn.  A sample is a point (Px, Py) of the 1/256 grid; pixel
// (px, py) owns the samples 256 px + [lo, hi] x 256 py + [lo, hi] (lo = hi = 128: the centre alone).
#pragma once
#include "common.cuh"

namespace icon {

constexpr unsigned long long RS_EMPTY = 0xffffffffffffffffull;
constexpr float RS_RANGE = 65536.f;          // |x_w|, |y_w| limit of the exact fixed-point path (pixels)

// one face, set up for coverage: internal corner order (0, 1, 2) or (0, 2, 1) so that the face is counter-clockwise
struct RsTri {
    int X[3], Y[3];      // internal order
    long long area;      // > 0
    bool swapped;
    int bx0, bx1, by0, by1;   // pixel box clamped to the viewport (empty when bx0 > bx1 or by0 > by1)
};

// the face of records r[3] (original corner order); false when it is not drawn (a record not ok, zero snapped area)
// or its pixel box misses the viewport
__device__ __forceinline__ bool rs_setup(const int4 r[3], int W, int H, int lo, int hi, RsTri &t) {
    if (!(r[0].w && r[1].w && r[2].w)) return false;
    long long area = (long long)(r[1].x - r[0].x) * (r[2].y - r[0].y) - (long long)(r[1].y - r[0].y) * (r[2].x - r[0].x);
    if (area == 0) return false;
    t.swapped = area < 0;
    t.area = t.swapped ? -area : area;
    const int4 ra = t.swapped ? r[2] : r[1], rb = t.swapped ? r[1] : r[2];
    t.X[0] = r[0].x; t.Y[0] = r[0].y; t.X[1] = ra.x; t.Y[1] = ra.y; t.X[2] = rb.x; t.Y[2] = rb.y;
    const int xmin = min(min(t.X[0], t.X[1]), t.X[2]), xmax = max(max(t.X[0], t.X[1]), t.X[2]);
    const int ymin = min(min(t.Y[0], t.Y[1]), t.Y[2]), ymax = max(max(t.Y[0], t.Y[1]), t.Y[2]);
    // pixels with a sample 256 p + [lo, hi] in [min, max]; >> is a floor division
    t.bx0 = max(-((hi - xmin) >> 8), 0); t.bx1 = min((xmax - lo) >> 8, W - 1);
    t.by0 = max(-((hi - ymin) >> 8), 0); t.by1 = min((ymax - lo) >> 8, H - 1);
    return t.bx0 <= t.bx1 && t.by0 <= t.by1;
}

// edge functions at (Px, Py) in INTERNAL order (edge k runs from corner k + 1 to k + 2); exact in int64
__device__ __forceinline__ void rs_edges(const RsTri &t, int Px, int Py, long long ei[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int a = (k + 1) % 3, b = (k + 2) % 3;
        ei[k] = (long long)(t.X[b] - t.X[a]) * (Py - t.Y[a]) - (long long)(t.Y[b] - t.Y[a]) * (Px - t.X[a]);
    }
}

// internal -> ORIGINAL corner order
__device__ __forceinline__ void rs_orig(const RsTri &t, const long long ei[3], long long e[3]) {
    e[0] = ei[0];
    e[1] = t.swapped ? ei[2] : ei[1];
    e[2] = t.swapped ? ei[1] : ei[2];
}

// edge functions at (Px, Py) by ORIGINAL corner; false when the point is not covered (top-left rule, y up)
__device__ __forceinline__ bool rs_cover(const RsTri &t, int Px, int Py, long long e[3]) {
    long long ei[3];
    rs_edges(t, Px, Py, ei);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int a = (k + 1) % 3, b = (k + 2) % 3;
        const int dx = t.X[b] - t.X[a], dy = t.Y[b] - t.Y[a];
        const bool top_left = dy < 0 || (dy == 0 && dx < 0);
        if (ei[k] < 0 || (ei[k] == 0 && !top_left)) return false;
    }
    rs_orig(t, ei, e);
    return true;
}

__device__ __forceinline__ void rs_weights(const RsTri &t, const long long e[3], float l[3]) {
    const float fa = __ll2float_rn(t.area);
#pragma unroll
    for (int k = 0; k < 3; ++k) l[k] = __ll2float_rn(e[k]) / fa;
}

// depth key of a fragment at interpolated window depth z: false when it is clipped (z outside [0, 1]) or cannot pass
// GL_LESS against the cleared 24-bit depth; else (q << 32 | face), nearest q then lowest face first
__device__ __forceinline__ bool rs_depth_key(float z, int f, unsigned long long &key) {
    if (!(z >= 0.f && z <= 1.f)) return false;
    const unsigned q = (unsigned)rintf(z * 16777215.f);
    if (q >= 16777215u) return false;
    key = ((unsigned long long)q << 32) | (unsigned)f;
    return true;
}

}  // namespace icon
