// nms.cu -- rotated-BEV IoU and greedy NMS on the device.
//   open3d.ml.torch.ops.nms(boxes [N,5] (x0, y0, x1, y1, r), scores [N], thr) -> int64 keep indices
//       call site: ml3d/torch/utils/objdet_helper.py:316-350 (multiclass_nms) <- Anchor3DHead.get_bboxes_single
//       (ml3d/torch/models/point_pillars.py:967-1025)
//   open3d.ml.contrib.iou_bev_{cpu,cuda}(a [N,5] (x, y, w, h, r), b [M,5]) -> [N,M]
//   open3d.ml.contrib.iou_3d_{cpu,cuda}(a [N,7] (x, y, z, w, h, l, ry), b [M,7]) -> [N,M]
//       call sites: ml3d/metrics/mAP.py:85-89, ml3d/datasets/utils/operations.py:430
// Contract (upstream Open3D is not vendored: parity unpinned, oracle/ops_ref.c restates the same):
//   * a box is the rectangle centre (cx, cy), size (w, h) rotated by r about its centre; the overlap of two
//     boxes is the area of the intersection polygon (Sutherland-Hodgman clipping, shoelace area) in fp32;
//   * nms: boxes are visited by descending score (ties: lower index first); a box is kept unless its IoU with an
//     already kept box exceeds thr; the result lists the kept ORIGINAL indices in visiting order;
//   * iou_3d: (x, z) is the ground plane with footprint (w, l) and heading ry, y the vertical axis with the box
//     spanning [y - h, y] (KITTI camera frame, the layout of pred['bbox'] in mAP.py).
// Integer / latency-bound work: one sort, one all-pairs pass (N^2 / 2 IoUs, 20 B per box read), one sequential
// greedy sweep over the suppression bit matrix by a single warp.
#include "../../include/o3dml_b200.h"
#include "prims.cuh"
#include "rbox.cuh"

namespace o3dml {

// ---- all-pairs IoU matrices ------------------------------------------------------------------------
// mode 0: bev [.,5] (x, y, w, h, r); mode 1: 3d [.,7] (x, y, z, w, h, l, ry)
__global__ void iou_matrix_kernel(const float* __restrict__ a, int64_t na, const float* __restrict__ b, int64_t nb,
                                  int mode, float* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= na * nb) return;
    const int64_t i = t / nb, j = t - i * nb;
    if (mode == 0) {
        const float* p = a + i * 5;
        const float* q = b + j * 5;
        out[t] = rbox_iou(rbox_xywhr(p[0], p[1], p[2], p[3], p[4]), rbox_xywhr(q[0], q[1], q[2], q[3], q[4]));
    } else {
        const float* p = a + i * 7;
        const float* q = b + j * 7;
        const RBox ra = rbox_xywhr(p[0], p[2], p[3], p[5], p[6]), rb = rbox_xywhr(q[0], q[2], q[3], q[5], q[6]);
        const float inter2 = rbox_intersection(ra, rb);
        const float ymax = fminf(p[1], q[1]), ymin = fmaxf(p[1] - p[4], q[1] - q[4]);
        const float ih = fmaxf(ymax - ymin, 0.f);
        const float inter = inter2 * ih;
        const float uni = p[3] * p[4] * p[5] + q[3] * q[4] * q[5] - inter;
        out[t] = uni > 0.f ? inter / uni : 0.f;
    }
}

// ---- NMS ---------------------------------------------------------------------------------------------
__global__ void nms_keys_kernel(const float* __restrict__ scores, int64_t n, uint64_t* __restrict__ keys) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t u = __float_as_uint(scores[i]);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);    // ascending order of u == ascending order of the float
    keys[i] = (uint64_t)(~u);                          // descending score
}

// mask[i][jb] bit k = IoU(sorted i, sorted jb*64 + k) > thr, only for j > i
__global__ void nms_mask_kernel(const float* __restrict__ boxes, const uint32_t* __restrict__ order, int64_t n, float thr,
                                uint64_t* __restrict__ mask, int64_t words) {
    const int64_t ib = blockIdx.y, jb = blockIdx.x;
    if (jb < ib) return;
    __shared__ float sb[64][5];
    const int64_t j0 = jb * 64;
    if (j0 + threadIdx.x < n) {
        const float* q = boxes + (size_t)order[j0 + threadIdx.x] * 5;
#pragma unroll
        for (int k = 0; k < 5; ++k) sb[threadIdx.x][k] = q[k];
    }
    __syncthreads();
    const int64_t i = ib * 64 + threadIdx.x;
    if (i >= n) return;
    const float* p = boxes + (size_t)order[i] * 5;
    const RBox a = rbox_xywhr(0.5f * (p[0] + p[2]), 0.5f * (p[1] + p[3]), p[2] - p[0], p[3] - p[1], p[4]);
    uint64_t bits = 0;
    const int cnt = (int)min((int64_t)64, n - j0);
    for (int k = (ib == jb ? threadIdx.x + 1 : 0); k < cnt; ++k) {
        const RBox b = rbox_xywhr(0.5f * (sb[k][0] + sb[k][2]), 0.5f * (sb[k][1] + sb[k][3]), sb[k][2] - sb[k][0],
                                  sb[k][3] - sb[k][1], sb[k][4]);
        if (rbox_iou(a, b) > thr) bits |= 1ull << k;
    }
    mask[i * words + jb] = bits;
}

// one warp: sequential sweep over the sorted boxes, suppression bits accumulated in shared memory
__global__ void nms_sweep_kernel(const uint64_t* __restrict__ mask, const uint32_t* __restrict__ order, int64_t n,
                                 int64_t words, int64_t* __restrict__ keep, int64_t* __restrict__ num_keep) {
    extern __shared__ uint64_t remv[];
    for (int64_t w = threadIdx.x; w < words; w += 32) remv[w] = 0;
    __syncwarp();
    int64_t kept = 0;
    for (int64_t i = 0; i < n; ++i) {
        const int64_t wi = i >> 6;
        const bool dead = (remv[wi] >> (i & 63)) & 1ull;
        if (!dead) {
            if (threadIdx.x == 0) keep[kept] = (int64_t)order[i];
            ++kept;
            for (int64_t w = wi + threadIdx.x; w < words; w += 32) remv[w] |= mask[i * words + w];
        }
        __syncwarp();
    }
    if (threadIdx.x == 0) *num_keep = kept;
}

// the sort of the scores, then the [n][words] suppression bit matrix
static std::pair<RadixSortBufs, uint64_t*> nms_carve(Workspace& ws, int64_t n) {
    n = n > 0 ? n : 1;
    const RadixSortBufs sort = radix_sort_carve(ws, n);
    return {sort, ws.take<uint64_t>((size_t)n * ceil_div<int64_t>(n, 64))};
}

}  // namespace o3dml

using namespace o3dml;

extern "C" size_t o3dml_nms_workspace_bytes(int64_t num_boxes) { return Workspace::measure(nms_carve, num_boxes); }

extern "C" int o3dml_nms(const float* boxes, const float* scores, int64_t num_boxes, float iou_threshold,
                         int64_t* keep_indices, int64_t* d_num_keep, void* workspace, size_t workspace_bytes,
                         void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(num_boxes >= 0, "nms: bad arguments");
    if (num_boxes == 0) {
        O3DML_CHECK(d_num_keep, "nms: bad arguments");
        O3DML_CUDA(cudaMemsetAsync(d_num_keep, 0, sizeof(int64_t), st));
        return O3DML_OK;
    }
    O3DML_CHECK(num_boxes <= 65536, "nms: at most 65 536 boxes (the suppression matrix is N^2 / 8 bytes)");
    const int64_t n = num_boxes, words = ceil_div<int64_t>(n, 64);
    O3DML_CHECK(words * 8 <= 48 * 1024, "nms: too many boxes for the sweep kernel");
    Workspace ws(workspace, workspace_bytes);
    auto [sort, mask] = nms_carve(ws, n);
    O3DML_CHECK_WORKSPACE(ws, "nms");
    O3DML_CHECK(d_num_keep, "nms: bad arguments");
    O3DML_CHECK(boxes && scores && keep_indices, "nms: null input");
    O3DML_CUDA(launch<nms_keys_kernel>((unsigned)ceil_div<int64_t>(n, 256), 256, 0, st, scores, n, sort.keys_a));
    O3DML_CUDA(radix_sort_pairs(sort, true, n, 32, st));
    const uint32_t* order = sort.vals_a;
    O3DML_CUDA(cudaMemsetAsync(mask, 0, (size_t)n * words * 8, st));
    dim3 grid((unsigned)words, (unsigned)words);
    O3DML_CUDA(launch<nms_mask_kernel>(grid, 64, 0, st, boxes, order, n, iou_threshold, mask, words));
    O3DML_CUDA(launch<nms_sweep_kernel>(1, 32, (size_t)words * 8, st, mask, order, n, words, keep_indices, d_num_keep));
    return O3DML_OK;
}

extern "C" int o3dml_iou_matrix(const float* boxes_a, int64_t num_a, const float* boxes_b, int64_t num_b, int mode,
                                float* out, void* stream) {
    O3DML_CHECK(mode == 0 || mode == 1, "iou: mode 0 (bev, [.,5]) or 1 (3d, [.,7])");
    if (num_a <= 0 || num_b <= 0) return O3DML_OK;
    O3DML_CHECK(boxes_a && boxes_b && out, "iou: null input");
    O3DML_CUDA(launch<iou_matrix_kernel>((unsigned)ceil_div<int64_t>(num_a * num_b, 128), 128, 0, (cudaStream_t)stream,
                                         boxes_a, num_a, boxes_b, num_b, mode, out));
    return O3DML_OK;
}
