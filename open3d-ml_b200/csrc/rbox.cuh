// rbox.cuh -- rotated-rectangle overlap in fp32, shared by the NMS op (nms.cu) and the fused detection
// post-processing (detect.cu), so that both decide "IoU > thr" with the same arithmetic.
//   A box is the rectangle centre (cx, cy), size (w, h) rotated by r about its centre; the overlap of two boxes
//   is the area of the intersection polygon (Sutherland-Hodgman clipping, shoelace area).
#pragma once
#include <cuda_runtime.h>

namespace o3dml {

struct RBox {
    float cx, cy, w, h, c, s;
};

__device__ __forceinline__ RBox rbox_xywhr(float cx, float cy, float w, float h, float r) {
    RBox b;
    b.cx = cx; b.cy = cy; b.w = w; b.h = h;
    sincosf(r, &b.s, &b.c);
    return b;
}

// the nms contract's (x0, y0, x1, y1, r) form
__device__ __forceinline__ RBox rbox_xyxyr(const float* p) {
    return rbox_xywhr(0.5f * (p[0] + p[2]), 0.5f * (p[1] + p[3]), p[2] - p[0], p[3] - p[1], p[4]);
}

__device__ __forceinline__ void rbox_corners(const RBox& b, float* x, float* y) {
    const float hw = 0.5f * b.w, hh = 0.5f * b.h;
    const float dx[4] = {-hw, hw, hw, -hw}, dy[4] = {-hh, -hh, hh, hh};   // counter-clockwise
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        x[i] = b.cx + dx[i] * b.c - dy[i] * b.s;
        y[i] = b.cy + dx[i] * b.s + dy[i] * b.c;
    }
}

// area of (rectangle a) intersect (rectangle b): clip a's polygon by b's four half-planes
static __device__ float rbox_intersection(const RBox& a, const RBox& b) {
    if (!(a.w > 0.f) || !(a.h > 0.f) || !(b.w > 0.f) || !(b.h > 0.f)) return 0.f;
    float px[8], py[8], qx[8], qy[8];
    int n = 4;
    rbox_corners(a, px, py);
    float bx[4], by[4];
    rbox_corners(b, bx, by);
#pragma unroll 1
    for (int e = 0; e < 4 && n > 0; ++e) {
        const float x0 = bx[e], y0 = by[e], ex = bx[(e + 1) & 3] - x0, ey = by[(e + 1) & 3] - y0;
        int m = 0;
        float sx = px[n - 1], sy = py[n - 1];
        float sd = ex * (sy - y0) - ey * (sx - x0);     // >= 0: inside (left of the ccw edge)
        for (int i = 0; i < n; ++i) {
            const float tx = px[i], ty = py[i];
            const float td = ex * (ty - y0) - ey * (tx - x0);
            if ((sd >= 0.f) != (td >= 0.f)) {
                const float t = sd / (sd - td);
                if (m < 8) { qx[m] = sx + t * (tx - sx); qy[m] = sy + t * (ty - sy); ++m; }
            }
            if (td >= 0.f && m < 8) { qx[m] = tx; qy[m] = ty; ++m; }
            sx = tx; sy = ty; sd = td;
        }
        n = m;
        for (int i = 0; i < n; ++i) { px[i] = qx[i]; py[i] = qy[i]; }
    }
    if (n < 3) return 0.f;
    float area = 0.f;
    for (int i = 0; i < n; ++i) {
        const int j = (i + 1 == n) ? 0 : i + 1;
        area += px[i] * py[j] - px[j] * py[i];
    }
    return fmaxf(0.5f * area, 0.f);
}

__device__ __forceinline__ float rbox_iou(const RBox& a, const RBox& b) {
    const float inter = rbox_intersection(a, b);
    const float uni = a.w * a.h + b.w * b.h - inter;
    return uni > 0.f ? inter / uni : 0.f;
}

}  // namespace o3dml
