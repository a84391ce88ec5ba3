// detect.cu -- PointPillars box decoding on the device: the batched replacement of Anchor3DHead.get_bboxes
//   (ml3d/torch/models/point_pillars.py:945-1025 with multiclass_nms, objdet_helper.py:316-350).
// Contract: DESIGN.md section 2 ("PointPillars box decoding").  Per frame, rows r = (y * W + x) * A + a:
//   1. score_c(r) = sigmoid(cls[a * C + c, y, x]) in fp32 (accurate expf);
//   2. when N = H * W * A > nms_pre, keep the nms_pre rows of largest max_c score_c, ordered by (score descending,
//      row ascending); otherwise keep all rows in row order.  K = min(nms_pre, N);
//   3. BBoxCoder.decode of the kept rows against the cached anchors; direction = argmax of the two logits (ties: 0);
//   4. per class: kept rows with score_c > score_thr, greedy rotated-BEV NMS at IoU 0.01 (the constant of
//      objdet_helper.py:346) with the nms op's rules (rbox.cuh, visiting by descending score_c, ties by position in
//      the step-2 order, suppressed when IoU > 0.01);
//   5. output per frame: class 0's survivors in visiting order, then class 1's, ...; yaw corrected with
//      limit_period(yaw - dir_offset, 1, pi) + dir_offset + pi * dir (point_pillars.py:1020-1023), padded to C * K
//      rows (zeros, label -1).
// Launches (independent of B and C): top-k by a 5-pass radix select on the unique 55-bit key
// (score bits << 23 | (2^23 - 1 - row)) -- one memset + 6 launches, skipped when N <= nms_pre -- then sort + decode,
// per-class segment sort, suppression matrix, sweep and output: 5 launches.  No host synchronisation, no allocation.
#include <algorithm>

#include "../../include/o3dml_b200.h"
#include "common.cuh"
#include "rbox.cuh"

namespace o3dml {
namespace {

constexpr int kDigitBits = 11, kBins = 1 << kDigitBits, kPasses = 5;   // 5 x 11 = 55 key bits
constexpr int kRowBits = 23;
constexpr uint32_t kRowMask = (1u << kRowBits) - 1;
constexpr int kMaxK = 4096;                      // bitonic sort of K 64-bit keys in shared memory, 64 mask words
constexpr int kSelThreads = 256, kSelRows = 16384;
constexpr int kSortThreads = 1024;
constexpr float kNmsIou = 0.01f;                 // objdet_helper.py:346, not the head's (training-only) iou_thr
constexpr float kPi = 3.14159265358979323846f;  // np.pi as fp32, as torch applies a Python float to a float32 tensor

struct SelState {
    unsigned long long prefix, thr;   // key bits resolved so far; selection threshold once done
    int need, done;                   // rows still to take inside the prefix
};

__device__ __forceinline__ float pp_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ int pass_shift(int p) { return kDigitBits * (kPasses - 1 - p); }

// Resolves one radix pass for the block's frame: the digit d whose bin holds the need-th largest key in the prefix.
// kSelThreads threads, each owning 8 consecutive digits (thread 0 the highest).
__device__ void resolve_pass(const uint32_t* __restrict__ h, SelState& st, int shift) {
    __shared__ uint32_t part[kSelThreads];
    __shared__ SelState res;
    if (st.done) return;                                    // uniform over the block
    const int t = threadIdx.x;
    uint32_t v[8], loc = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) { v[q] = h[kBins - 1 - 8 * t - q]; loc += v[q]; }
    part[t] = loc;
    __syncthreads();
    for (int off = 1; off < kSelThreads; off <<= 1) {
        const uint32_t x = t >= off ? part[t - off] : 0u;
        __syncthreads();
        part[t] += x;
        __syncthreads();
    }
    const uint32_t need = (uint32_t)st.need;
    uint32_t cum = part[t] - loc;
    if (cum < need && need <= part[t]) {
        for (int q = 0; q < 8; ++q) {
            if (cum + v[q] >= need) {
                const uint32_t d = kBins - 1 - 8 * t - q;
                res.need = (int)(need - cum);
                res.prefix = (st.prefix << kDigitBits) | d;
                res.done = (v[q] == need - cum || shift == 0) ? 1 : 0;
                res.thr = res.prefix << shift;
                break;
            }
            cum += v[q];
        }
    }
    __syncthreads();
    st = res;
}

// pass 0: scores -> keys32 + histogram of digit 0; pass 1..4: resolve pass - 1, histogram of digit `pass` inside the
// prefix; pass 5: resolve pass 4 and write the K selected keys (any order) to cand.
// Element t of a frame is (a = t / HW, pos = t % HW): consecutive threads read consecutive pixels of one channel.
__global__ void __launch_bounds__(kSelThreads) pp_select_kernel(
    int pass, const float* __restrict__ cls, int64_t cls_bs, int HW, int A, int C, int64_t N, int K,
    uint32_t* __restrict__ keys32, uint32_t* __restrict__ hist, SelState* __restrict__ states,
    int* __restrict__ cand_count, unsigned long long* __restrict__ cand) {
    const int B = gridDim.y, b = blockIdx.y;
    __shared__ uint32_t sh[kBins];
    SelState st;
    if (pass <= 1) { st.prefix = 0; st.thr = 0; st.need = K; st.done = 0; }
    else st = states[(size_t)(pass - 2) * B + b];
    if (pass >= 1) {
        resolve_pass(hist + ((size_t)(pass - 1) * B + b) * kBins, st, pass_shift(pass - 1));
        if (blockIdx.x == 0 && threadIdx.x == 0) states[(size_t)(pass - 1) * B + b] = st;
        if (pass < kPasses && st.done) return;
    }
    const int64_t t0 = (int64_t)blockIdx.x * kSelRows, t1 = min(N, t0 + kSelRows);
    uint32_t* k32 = keys32 + (size_t)b * N;
    if (pass == kPasses) {
        for (int64_t t = t0 + threadIdx.x; t < t1; t += kSelThreads) {
            const uint32_t row = (uint32_t)((t % HW) * A + t / HW);
            const unsigned long long key = ((unsigned long long)k32[t] << kRowBits) | (kRowMask - row);
            if (key >= st.thr) {
                const int slot = atomicAdd(cand_count + b, 1);
                if (slot < K) cand[(size_t)b * K + slot] = key;
            }
        }
        return;
    }
    for (int i = threadIdx.x; i < kBins; i += kSelThreads) sh[i] = 0;
    __syncthreads();
    const int shift = pass_shift(pass);
    for (int64_t t = t0 + threadIdx.x; t < t1; t += kSelThreads) {
        const int a = (int)(t / HW), pos = (int)(t % HW);
        uint32_t sbits;
        if (pass == 0) {
            const float* p = cls + (size_t)b * cls_bs + (size_t)a * C * HW + pos;
            float m = p[0];
            for (int c = 1; c < C; ++c) m = fmaxf(m, p[(size_t)c * HW]);
            sbits = __float_as_uint(pp_sigmoid(m));     // sigmoid is monotone: max of sigmoids = sigmoid of the max
            k32[t] = sbits;
        } else {
            sbits = k32[t];
        }
        const uint32_t row = (uint32_t)pos * A + a;
        const unsigned long long key = ((unsigned long long)sbits << kRowBits) | (kRowMask - row);
        if (pass == 0 || (key >> (shift + kDigitBits)) == st.prefix)
            atomicAdd(&sh[(key >> shift) & (kBins - 1)], 1u);
    }
    __syncthreads();
    uint32_t* hg = hist + ((size_t)pass * B + b) * kBins;
    for (int i = threadIdx.x; i < kBins; i += kSelThreads)
        if (sh[i]) atomicAdd(hg + i, sh[i]);
}

// descending bitonic sort of n (a power of two) keys in shared memory
__device__ void bitonic_sort_desc(unsigned long long* s, int n) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = s[i], y = s[ixj];
                    const bool desc = (i & k) == 0;
                    if (desc ? x < y : x > y) { s[i] = y; s[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
}

// one block per frame: the top-k order (or row order), then decode of the K kept rows.
// BBoxCoder.decode (objdet_helper.py:287-313) with every product and sum rounded on its own, as torch computes it.
__global__ void __launch_bounds__(kSortThreads) pp_topk_decode_kernel(
    const unsigned long long* __restrict__ cand, int select, int K, int P, const float* __restrict__ cls, int64_t cls_bs,
    const float* __restrict__ reg, int64_t reg_bs, const float* __restrict__ dirm, int64_t dir_bs, int HW, int A, int C,
    const float* __restrict__ anchors, float* __restrict__ dec, int* __restrict__ dirc, float* __restrict__ sc) {
    extern __shared__ unsigned long long sk[];
    const int b = blockIdx.x;
    if (select) {
        for (int i = threadIdx.x; i < P; i += blockDim.x) sk[i] = i < K ? cand[(size_t)b * K + i] : 0ull;
        __syncthreads();
        bitonic_sort_desc(sk, P);
    }
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        const uint32_t row = select ? kRowMask - (uint32_t)(sk[i] & kRowMask) : (uint32_t)i;
        const int a = (int)(row % A), pos = (int)(row / A);
        const float* an = anchors + (size_t)row * 7;
        const float* dl = reg + (size_t)b * reg_bs + (size_t)a * 7 * HW + pos;
        const float xa = an[0], ya = an[1], wa = an[3], la = an[4], ha = an[5];
        const float za = __fadd_rn(an[2], __fmul_rn(ha, 0.5f));
        const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
        float* o = dec + ((size_t)b * K + i) * 7;
        const float hg = __fmul_rn(expf(dl[5 * HW]), ha);
        o[0] = __fadd_rn(__fmul_rn(dl[0], diag), xa);
        o[1] = __fadd_rn(__fmul_rn(dl[HW], diag), ya);
        o[2] = __fsub_rn(__fadd_rn(__fmul_rn(dl[2 * HW], ha), za), __fmul_rn(hg, 0.5f));
        o[3] = __fmul_rn(expf(dl[3 * HW]), wa);
        o[4] = __fmul_rn(expf(dl[4 * HW]), la);
        o[5] = hg;
        o[6] = __fadd_rn(dl[6 * HW], an[6]);
        const float* dp = dirm + (size_t)b * dir_bs + (size_t)a * 2 * HW + pos;
        dirc[(size_t)b * K + i] = dp[HW] > dp[0] ? 1 : 0;
        const float* cp = cls + (size_t)b * cls_bs + (size_t)a * C * HW + pos;
        for (int c = 0; c < C; ++c) sc[((size_t)b * K + i) * C + c] = pp_sigmoid(cp[(size_t)c * HW]);
    }
}

// one block per (frame, class): the kept rows above score_thr by (score_c descending, position ascending), and their
// BEV boxes (x - w/2, y - l/2, x + w/2, y + l/2, r) (objdet_helper.py:69-99)
__global__ void __launch_bounds__(kSortThreads) pp_class_sort_kernel(
    const float* __restrict__ sc, const float* __restrict__ dec, int K, int P, int C, float score_thr,
    int* __restrict__ seg_idx, float* __restrict__ bev, int* __restrict__ seg_cnt) {
    extern __shared__ unsigned long long sk[];
    __shared__ int cnt;
    const int seg = blockIdx.x, b = seg / C, c = seg - b * C;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        unsigned long long key = 0;
        if (i < K) {
            const float s = sc[((size_t)b * K + i) * C + c];
            if (s > score_thr) {
                key = ((unsigned long long)__float_as_uint(s) << 32) | (0xFFFFFFFFu - (uint32_t)i);
                atomicAdd(&cnt, 1);
            }
        }
        sk[i] = key;
    }
    __syncthreads();
    bitonic_sort_desc(sk, P);
    const int m = cnt;
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
        const int k = (int)(0xFFFFFFFFu - (uint32_t)(sk[j] & 0xFFFFFFFFull));
        seg_idx[(size_t)seg * K + j] = k;
        const float* d = dec + ((size_t)b * K + k) * 7;
        const float hw = d[3] / 2.f, hl = d[4] / 2.f;
        float* q = bev + ((size_t)seg * K + j) * 5;
        q[0] = d[0] - hw; q[1] = d[1] - hl; q[2] = d[0] + hw; q[3] = d[1] + hl; q[4] = d[6];
    }
    if (threadIdx.x == 0) seg_cnt[seg] = m;
}

// suppression matrix of every segment in one grid (x: column block, y: row block, z: segment).  Pairs whose
// bounding circles are disjoint (with a margin far above fp32 rounding) have IoU exactly 0 <= thr: no clipping.
__global__ void __launch_bounds__(64) pp_nms_mask_kernel(const float* __restrict__ bev, const int* __restrict__ seg_cnt,
                                                         int K, int words_max, unsigned long long* __restrict__ mask) {
    const int seg = blockIdx.z, ib = blockIdx.y, jb = blockIdx.x;
    const int n = seg_cnt[seg], words = (n + 63) >> 6;
    if (jb < ib || jb >= words) return;
    __shared__ RBox sb[64];
    __shared__ float sr[64];
    const float* base = bev + (size_t)seg * K * 5;
    const int j0 = jb * 64;
    if (j0 + (int)threadIdx.x < n) {
        const RBox q = rbox_xyxyr(base + (size_t)(j0 + threadIdx.x) * 5);
        sb[threadIdx.x] = q;
        sr[threadIdx.x] = 0.5f * sqrtf(q.w * q.w + q.h * q.h);
    }
    __syncthreads();
    const int i = ib * 64 + threadIdx.x;
    if (i >= n) return;
    const RBox a = rbox_xyxyr(base + (size_t)i * 5);
    const float ra = 0.5f * sqrtf(a.w * a.w + a.h * a.h);
    unsigned long long bits = 0;
    const int cnt = min(64, n - j0);
    for (int k = (ib == jb ? threadIdx.x + 1 : 0); k < cnt; ++k) {
        const float dx = a.cx - sb[k].cx, dy = a.cy - sb[k].cy, rr = 1.001f * (ra + sr[k]) + 1e-6f;
        if (dx * dx + dy * dy > rr * rr) continue;
        if (rbox_iou(a, sb[k]) > kNmsIou) bits |= 1ull << k;
    }
    mask[((size_t)seg * K + i) * words_max + jb] = bits;
}

// one warp per segment: the greedy sweep of nms.cu over the segment's bit matrix
__global__ void __launch_bounds__(32) pp_nms_sweep_kernel(const unsigned long long* __restrict__ mask,
                                                          const int* __restrict__ seg_idx, const int* __restrict__ seg_cnt,
                                                          int K, int words_max, int* __restrict__ keep,
                                                          int* __restrict__ nkeep) {
    __shared__ unsigned long long remv[kMaxK / 64];
    const int seg = blockIdx.x, n = seg_cnt[seg], words = (n + 63) >> 6;
    for (int w = threadIdx.x; w < words; w += 32) remv[w] = 0;
    __syncwarp();
    const unsigned long long* m = mask + (size_t)seg * K * words_max;
    int kept = 0;
    for (int i = 0; i < n; ++i) {
        const int wi = i >> 6;
        if (!((remv[wi] >> (i & 63)) & 1ull)) {
            if (threadIdx.x == 0) keep[(size_t)seg * K + kept] = seg_idx[(size_t)seg * K + i];
            ++kept;
            for (int w = wi + threadIdx.x; w < words; w += 32) remv[w] |= m[(size_t)i * words_max + w];
        }
        __syncwarp();
    }
    if (threadIdx.x == 0) nkeep[seg] = kept;
}

// padded per-frame output: class offsets, yaw correction, zero fill with label -1
__global__ void pp_output_kernel(const float* __restrict__ dec, const int* __restrict__ dirc, const float* __restrict__ sc,
                                 const int* __restrict__ keep, const int* __restrict__ nkeep, int K, int C,
                                 float dir_offset, float* __restrict__ out_boxes, float* __restrict__ out_scores,
                                 int64_t* __restrict__ out_labels, int64_t* __restrict__ counts) {
    const int b = blockIdx.y;
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t width = (int64_t)C * K;
    int c = -1, i = 0, total = 0;
    for (int q = 0; q < C; ++q) {
        const int n = nkeep[b * C + q];
        if (c < 0 && j < total + n) { c = q; i = (int)(j - total); }
        total += n;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) counts[b] = total;
    if (j >= width) return;
    float* ob = out_boxes + ((size_t)b * width + j) * 7;
    if (c < 0) {
        for (int q = 0; q < 7; ++q) ob[q] = 0.f;
        out_scores[(size_t)b * width + j] = 0.f;
        out_labels[(size_t)b * width + j] = -1;
        return;
    }
    const int k = keep[((size_t)b * C + c) * K + i];
    const float* d = dec + ((size_t)b * K + k) * 7;
    for (int q = 0; q < 6; ++q) ob[q] = d[q];
    // limit_period(yaw - off, 1, pi) + off + pi * dir, each operation rounded on its own (point_pillars.py:1021-1023)
    const float v = __fsub_rn(d[6], dir_offset);
    const float rot = __fsub_rn(v, __fmul_rn(floorf(__fadd_rn(__fdiv_rn(v, kPi), 1.f)), kPi));
    ob[6] = __fadd_rn(__fadd_rn(rot, dir_offset), __fmul_rn(kPi, (float)dirc[(size_t)b * K + k]));
    out_scores[(size_t)b * width + j] = sc[((size_t)b * K + k) * C + c];
    out_labels[(size_t)b * width + j] = c;
}

struct DetectBuffers {
    uint32_t* keys32;
    uint32_t* hist;
    int* cand_count;
    SelState* states;
    unsigned long long* cand;
    float *dec, *sc, *bev;
    int *dirc, *seg_idx, *seg_cnt, *keep, *nkeep;
    unsigned long long* mask;
};

DetectBuffers carve(Workspace& ws, int64_t B, int64_t N, int64_t K, int64_t C, bool select) {
    DetectBuffers d{};
    const int64_t words_max = (K + 63) / 64;
    if (select) {
        d.keys32 = ws.take<uint32_t>((size_t)(B * N));
        // hist and cand_count are adjacent: one memset clears both
        d.hist = ws.take<uint32_t>((size_t)(kPasses * B * kBins + B));
        d.cand_count = d.hist ? (int*)(d.hist + kPasses * B * kBins) : nullptr;
        d.states = ws.take<SelState>((size_t)(kPasses * B));
        d.cand = ws.take<unsigned long long>((size_t)(B * K));
    }
    d.dec = ws.take<float>((size_t)(B * K * 7));
    d.dirc = ws.take<int>((size_t)(B * K));
    d.sc = ws.take<float>((size_t)(B * K * C));
    d.seg_idx = ws.take<int>((size_t)(B * C * K));
    d.bev = ws.take<float>((size_t)(B * C * K * 5));
    d.seg_cnt = ws.take<int>((size_t)(B * C));
    d.mask = ws.take<unsigned long long>((size_t)(B * C * K * words_max));
    d.keep = ws.take<int>((size_t)(B * C * K));
    d.nkeep = ws.take<int>((size_t)(B * C));
    return d;
}

}  // namespace
}  // namespace o3dml

using namespace o3dml;

static int detect_check(int64_t batch, int64_t height, int64_t width, int num_anchors, int num_classes,
                        int64_t nms_pre) {
    O3DML_CHECK(batch >= 0 && height >= 1 && width >= 1 && num_anchors >= 1 && num_classes >= 1,
                "pp_detect: bad shape");
    O3DML_CHECK(nms_pre >= 1 && nms_pre <= kMaxK, "pp_detect: nms_pre must be in [1, %d] (got %lld)", kMaxK,
                (long long)nms_pre);
    O3DML_CHECK(height * width * num_anchors <= (int64_t)kRowMask - 1, "pp_detect: at most %u rows per frame",
                kRowMask - 1);
    O3DML_CHECK(batch * num_classes <= 65535, "pp_detect: batch * num_classes must not exceed 65535");
    return O3DML_OK;
}

extern "C" size_t o3dml_pp_detect_workspace_bytes(int64_t batch, int64_t height, int64_t width, int num_anchors,
                                                  int num_classes, int64_t nms_pre) {
    if (detect_check(batch, height, width, num_anchors, num_classes, nms_pre) != O3DML_OK) return 0;
    const int64_t N = height * width * num_anchors, K = std::min<int64_t>(nms_pre, N);
    return Workspace::measure(carve, batch, N, K, num_classes, N > nms_pre);
}

extern "C" int o3dml_pp_detect(const float* cls, int64_t cls_batch_stride, const float* reg, int64_t reg_batch_stride,
                               const float* dir, int64_t dir_batch_stride, int64_t batch, int64_t height, int64_t width,
                               int num_anchors, int num_classes, const float* anchors, int64_t nms_pre, float score_thr,
                               float dir_offset, float* out_boxes, float* out_scores, int64_t* out_labels,
                               int64_t* d_counts, void* workspace, size_t workspace_bytes, void* stream) {
    const int rc = detect_check(batch, height, width, num_anchors, num_classes, nms_pre);
    if (rc != O3DML_OK) return rc;
    if (batch == 0) return O3DML_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int B = (int)batch, C = num_classes, A = num_anchors, HW = (int)(height * width);
    const int64_t N = (int64_t)HW * A;
    const int K = (int)std::min<int64_t>(nms_pre, N);
    const bool select = N > nms_pre;
    int P = 1;
    while (P < K) P <<= 1;
    const int words_max = (K + 63) / 64;
    Workspace ws(workspace, workspace_bytes);
    const DetectBuffers d = carve(ws, B, N, K, C, select);
    O3DML_CHECK_WORKSPACE(ws, "pp_detect");
    O3DML_CHECK(cls && reg && dir && anchors && out_boxes && out_scores && out_labels && d_counts,
                "pp_detect: null input");
    if (select) {
        O3DML_CUDA(cudaMemsetAsync(d.hist, 0, ((size_t)kPasses * B * kBins + B) * sizeof(uint32_t), st));
        const dim3 grid((unsigned)ceil_div<int64_t>(N, kSelRows), (unsigned)B);
        for (int pass = 0; pass <= kPasses; ++pass)
            O3DML_CUDA(launch<pp_select_kernel>(grid, kSelThreads, 0, st, pass, cls, cls_batch_stride, HW, A, C, N, K,
                                                d.keys32, d.hist, d.states, d.cand_count, d.cand));
    }
    const size_t sort_smem = (size_t)P * sizeof(unsigned long long);
    O3DML_CUDA(launch<pp_topk_decode_kernel>(B, kSortThreads, select ? sort_smem : 0, st, d.cand, select ? 1 : 0, K, P,
                                             cls, cls_batch_stride, reg, reg_batch_stride, dir, dir_batch_stride, HW,
                                             A, C, anchors, d.dec, d.dirc, d.sc));
    O3DML_CUDA(launch<pp_class_sort_kernel>(B * C, kSortThreads, sort_smem, st, d.sc, d.dec, K, P, C, score_thr,
                                            d.seg_idx, d.bev, d.seg_cnt));
    O3DML_CUDA(launch<pp_nms_mask_kernel>(dim3((unsigned)words_max, (unsigned)words_max, (unsigned)(B * C)), 64, 0, st,
                                          d.bev, d.seg_cnt, K, words_max, d.mask));
    O3DML_CUDA(launch<pp_nms_sweep_kernel>(B * C, 32, 0, st, d.mask, d.seg_idx, d.seg_cnt, K, words_max, d.keep,
                                           d.nkeep));
    O3DML_CUDA(launch<pp_output_kernel>(dim3((unsigned)ceil_div<int64_t>((int64_t)C * K, 256), (unsigned)B), 256, 0, st,
                                        d.dec, d.dirc, d.sc, d.keep, d.nkeep, K, C, dir_offset, out_boxes, out_scores,
                                        out_labels, d_counts));
    return O3DML_OK;
}
