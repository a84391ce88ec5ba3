// rbox.cuh -- rotated-rectangle overlap in fp32 and the greedy NMS launcher, shared by the NMS op (nms.cu) and the
// fused detection post-processing (detect.cu), so that both decide "IoU > thr" with the same kernels.
//   A box is the rectangle centre (cx, cy), size (w, h) rotated by r about its centre; the overlap of two boxes
//   is the area of the intersection polygon (Sutherland-Hodgman clipping, shoelace area).
//   The clipping runs in a frame centred on the first box: at LiDAR ranges (70 m) absolute corner coordinates carry
//   rounding of a few 1e-6 m and shoelace products of a few 1e-4 m^2, which is the whole area of a 2 cm box.  Two boxes
//   that overlap have centres (and corners) within a factor of 2 of each other where the coordinates are large, so
//   their differences are exact (Sterbenz); near the axes the coordinates, and their rounding, are small.
//   The intersection is clamped to the smaller area, so that 0 <= IoU <= 1 holds under fp32 rounding.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace o3dml {

// the (x, y, w, h, r) form: centre, size, cos / sin of the heading
struct RBox {
    float cx, cy, w, h, c, s;
};

// the nms contract's (x0, y0, x1, y1, r) form: the rectangle [x0, x1] x [y0, y1] rotated by r about its centre
struct RBoxXY {
    float x0, y0, x1, y1, c, s;
};

__device__ __forceinline__ RBox rbox_xywhr(float cx, float cy, float w, float h, float r) {
    RBox b;
    b.cx = cx; b.cy = cy; b.w = w; b.h = h;
    sincosf(r, &b.s, &b.c);
    return b;
}

__device__ __forceinline__ RBoxXY rbox_xyxyr(const float* p) {
    RBoxXY b;
    b.x0 = p[0]; b.y0 = p[1]; b.x1 = p[2]; b.y1 = p[3];
    sincosf(p[4], &b.s, &b.c);
    return b;
}

// b's centre relative to a's, from corner differences (exact where the coordinates are large and the boxes close)
__device__ __forceinline__ void rbox_offset(const RBoxXY& a, const RBoxXY& b, float& dx, float& dy) {
    dx = 0.5f * ((b.x0 - a.x0) + (b.x1 - a.x1));
    dy = 0.5f * ((b.y0 - a.y0) + (b.y1 - a.y1));
}

// a plain product: never contracted into an FMA, so that the clamp of rbox_intersection and the union of rbox_iou
// see the same rounded area
__device__ __forceinline__ float rbox_area(const RBox& b) { return __fmul_rn(b.w, b.h); }

// corners of b moved so that its centre is (ox, oy)
__device__ __forceinline__ void rbox_corners(const RBox& b, float ox, float oy, float* x, float* y) {
    const float hw = 0.5f * b.w, hh = 0.5f * b.h;
    const float dx[4] = {-hw, hw, hw, -hw}, dy[4] = {-hh, -hh, hh, hh};   // counter-clockwise
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        x[i] = ox + dx[i] * b.c - dy[i] * b.s;
        y[i] = oy + dx[i] * b.s + dy[i] * b.c;
    }
}

// area of (rectangle a) intersect (rectangle b), at most min(area a, area b): clip a's polygon by b's four
// half-planes in a frame centred on a
static __device__ float rbox_intersection(const RBox& a, const RBox& b) {
    if (!(a.w > 0.f) || !(a.h > 0.f) || !(b.w > 0.f) || !(b.h > 0.f)) return 0.f;
    float px[8], py[8], qx[8], qy[8];
    int n = 4;
    rbox_corners(a, 0.f, 0.f, px, py);
    float bx[4], by[4];
    rbox_corners(b, b.cx - a.cx, b.cy - a.cy, bx, by);
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
    return fminf(fmaxf(0.5f * area, 0.f), fminf(rbox_area(a), rbox_area(b)));
}

// inter <= min(area a, area b) makes fl(fl(area a + area b) - inter) >= inter under round-to-nearest: IoU <= 1
__device__ __forceinline__ float rbox_iou(const RBox& a, const RBox& b) {
    const float inter = rbox_intersection(a, b);
    const float uni = rbox_area(a) + rbox_area(b) - inter;
    return uni > 0.f ? inter / uni : 0.f;
}

// the (x0, y0, x1, y1, r) form, in a frame centred on a.  For degenerate boxes (km-long slivers) the fp32 result
// depends on FMA contraction, which shifts if the caller also computes these corner differences or this offset.
__device__ __forceinline__ float rbox_iou(const RBoxXY& a, const RBoxXY& b) {
    RBox ra, rb;
    ra.cx = 0.f; ra.cy = 0.f; ra.w = a.x1 - a.x0; ra.h = a.y1 - a.y0; ra.c = a.c; ra.s = a.s;
    rbox_offset(a, b, rb.cx, rb.cy);
    rb.w = b.x1 - b.x0; rb.h = b.y1 - b.y0; rb.c = b.c; rb.s = b.s;
    return rbox_iou(ra, rb);
}

// Greedy NMS of `segments` box lists in two launches (nms.cu).  Segment s visits ids[s * ids_stride + i] for i below
// counts[s] (n_max when counts is null), (x0, y0, x1, y1, r) rows of boxes + (s / segs_per_set) * set_stride, and
// writes the ids it keeps, in visiting order, to keep + s * keep_stride and their number to num_keep[s].
// mask: segments * n_max * ceil(n_max / 64) words of scratch, not cleared.  Out is int or int64_t.
template <typename Out>
cudaError_t nms_segments(const float* boxes, int64_t set_stride, int segs_per_set, const int* ids, int64_t ids_stride,
                         const int* counts, int n_max, int segments, float thr, uint64_t* mask, Out* keep,
                         int64_t keep_stride, Out* num_keep, cudaStream_t st);

}  // namespace o3dml
