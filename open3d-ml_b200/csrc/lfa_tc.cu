// lfa_tc.cu -- RandLA-Net attentive-pooling stage on the Hopper tensor cores (wgmma):
//   neighbour gather -> LocSE encoding (+ shared MLPs) -> score GEMM on the tensor cores with the
//   3xFP16 split (tc.cuh) -> softmax over the 16 neighbours -> weighted sum  ==> agg [N, d]
// Same contract as lfa_pool_kernel (lfa.cu); replaces randlanet.py:521-639 as used at :667-692.
//
// One tile = 128 neighbour rows = 8 points x 16 neighbours, 256 threads = two warpgroups of 64 rows:
//   A  [128 x d]  : X = [feat[nbr] | r1 or r2], built by the CTA in shared memory directly in the
//                   chunk-major layout (one conflict-free 16-byte store per (row, 8 channels)),
//                   as fp16 hi/lo pairs.  In stage 2 the first half of A first holds r1 (the A
//                   operand of the lse2 GEMM) and is then overwritten by the gathered features.
//   B  [d x d]    : score weight, host-packed hi/lo operand image; resident in shared memory for
//                   d <= 128, streamed for d = 256 through a ring of two 32-row column blocks filled by bulk
//                   copies (mbarrier completion), one tile's blocks after the other's
//   D             : CB score columns per block (64 for d = 64 / 128, 32 for d = 256, d below), each warpgroup's
//                   [64 x CB] block in registers; block j + 1 is issued into a second accumulator set before the
//                   epilogue of block j runs (wait_group 1)
// Epilogue on the accumulator registers: warp w of a warpgroup holds rows [16w, 16w + 16) = the 16 neighbours of one
// point, a thread rows g and g + 8 of its column pairs.  Column max and the sums of e and e.x over the 16 rows: the two
// rows in registers, then the 8 lanes sharing lane % 4 (max: butterfly; sums: reduce-scatter, so that the lanes store
// distinct columns of the point's agg row).  x = hi + lo is read from A at (row, column pair), one conflict-free 4-byte
// load per operand.
// Stage 2 chains a second GEMM (r2 = lrelu(BN(Wl2 . r1)), N = d/2) whose epilogue writes r2 from the registers into
// A (d = 16: that 8x8 product stays in registers).  The score bias is not applied: it is constant over the neighbours of
// a point and cancels in the softmax.  CTAs are persistent over tiles.  Two tiles are in flight per SM at d = 64 (two
// CTAs) and d = 128 (two A tiles in one CTA: tile t+1 is built while tile t's score MMAs run).
#include "../../include/o3dml_b200.h"
#include "common.cuh"
#include "tc.cuh"

namespace o3dml {

constexpr int LTC_ROWS = 128;  // MMA M
constexpr int LTC_K = 16;      // neighbours

struct LfaTcParams {
    const float* coords;
    const void* nidx;
    int nidx_is64;
    const float* feat;     // [B*N, D/2]
    int64_t total, n_per_batch;
    const float* w10t;     // [10][D/2]
    const float* s10;
    const float* t10;
    const uint4* wl2_img;  // stage 2, d >= 32: [hi | lo] operand images of Wl2 [N=D/2][K=D/2]
    const float* wl2t;     // stage 2, d == 16: fp32 [in][out]
    const float* s2;
    const float* t2;
    const uint4* ws_img;   // [hi | lo] operand images of the score weight [N=D][K=D]
    float* agg;            // [B*N, D]
    int64_t num_tiles;
};

template <int D, int STAGE>
struct LtcCfg {
    static constexpr int H = D / 2;
    static constexpr bool STREAM = D > 128;          // weights do not fit next to the A tile
    static constexpr bool MMA2 = STAGE == 2 && H >= 16;  // lse2 on the tensor core
    static constexpr int NTH = 256;                  // threads per CTA: two warpgroups
    static constexpr int NPART = NTH / LTC_ROWS;     // threads sharing one row
    // score columns per block: 64 where the weight is resident, 32 where it streams through the ring (two 64-column
    // slots would not fit next to the 128 KB A tile)
    static constexpr int CB = D < 64 ? D : (STREAM ? 32 : 64);
    static constexpr int NBLK = D / CB;
    static constexpr int CB2 = STREAM ? 32 : (H < 64 ? H : 64);  // lse2 columns per block
    static constexpr int A_BYTES = D / 8 * LTC_ROWS * 16;  // one of hi / lo
    static constexpr int SLOT_BYTES = D / 8 * CB * 16;     // one of hi / lo of one streamed column block
    static constexpr int B_BYTES = STREAM ? 2 * SLOT_BYTES : D / 8 * D * 16;  // per hi / lo; streamed: two ring slots
    static constexpr int B2_BYTES = MMA2 ? (STREAM ? H / 8 * CB2 * 16 : H / 8 * H * 16) : 0;
    static constexpr int W10_BYTES = 12 * H * 4;
    static constexpr int ST2_BYTES = STAGE == 2 ? (2 * H + (H < 16 ? H * H : 0)) * 4 : 0;
    // Two tiles in flight per SM, so that the SIMT build of one tile overlaps the score MMAs of the other: d = 64 as two
    // CTAs per SM (<= 128 registers), d = 128 as two A tiles in one CTA (the CTA builds tile t+1 into one while the
    // tensor core works on tile t in the other).  d = 256 has room for neither.
    static constexpr int MIN_CTAS = D == 64 ? 2 : 1;
    static constexpr bool DBUF = D == 128;
    static constexpr int NBUF = DBUF ? 2 : 1;
    static constexpr size_t SMEM = NBUF * 2 * A_BYTES + 2 * B_BYTES + 2 * B2_BYTES + W10_BYTES + ST2_BYTES + 16 + 128;
};

// Issues (does not wait for) the warpgroup's 64 rows of A[128 x K] times a block of CBN rows of B (both hi / lo,
// chunk-major) -> d[CBN / 2], as one committed wgmma group
template <int CBN, int K>
__device__ __forceinline__ void ltc_issue(float* d, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                          uint32_t b_lbo, int wg) {
    constexpr uint32_t A_LBO = LTC_ROWS * 16;
    a_hi += (uint32_t)wg * 64 * 16;
    a_lo += (uint32_t)wg * 64 * 16;
#pragma unroll
    for (int i = 0; i < CBN / 2; ++i) tc::fence_operand(d[i]);
    tc::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < K / 16; ++ks) {
        const uint64_t ah = tc::smem_desc(a_hi + ks * 2 * A_LBO, A_LBO, 128);
        const uint64_t al = tc::smem_desc(a_lo + ks * 2 * A_LBO, A_LBO, 128);
        const uint64_t bh = tc::smem_desc(b_hi + ks * 2 * b_lbo, b_lbo, 128);
        const uint64_t bl = tc::smem_desc(b_lo + ks * 2 * b_lbo, b_lbo, 128);
        tc::wgmma_f16_ss<CBN>(d, ah, bh, ks > 0);
        tc::wgmma_f16_ss<CBN>(d, ah, bl, 1u);
        tc::wgmma_f16_ss<CBN>(d, al, bh, 1u);
    }
    tc::wgmma_commit();
#pragma unroll
    for (int i = 0; i < CBN / 2; ++i) tc::fence_operand(d[i]);
}

// Waits until at most N of this warpgroup's wgmma groups are pending; d (the oldest group's accumulators) is then final
template <int N, int CNT>
__device__ __forceinline__ void ltc_wait(float* d) {
    tc::wgmma_wait<N>();
#pragma unroll
    for (int i = 0; i < CNT; ++i) tc::fence_operand(d[i]);
}

// One bulk copy (TMA) per (hi / lo, 8-row k chunk) of column block nb of a weight image [K/8][NIMG][8] (hi, then lo)
// into a ring slot [hi | lo] of [K/8][CBN][8] each, completing on bar.  Every thread of the CTA runs it and the lanes of
// the warp with `issuer` set issue the copies: the instructions are predicated rather than branched around, because a
// divergent branch while a wgmma group is in flight makes ptxas serialize the wgmma instructions.
template <int CBN, int K, int NIMG>
__device__ __forceinline__ void ltc_fill(uint8_t* slot, uint64_t* bar, const uint4* __restrict__ img, int nb, int lane,
                                         bool issuer) {
    constexpr uint32_t ROW = CBN * 16, HALF = K / 8 * ROW;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t"
                 "@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(tc::smem_u32(bar)),
                 "r"(2 * HALF), "r"((int)(issuer && lane == 0))
                 : "memory");
#pragma unroll
    for (int i0 = 0; i0 < 2 * (K / 8); i0 += 32) {
        const int i = i0 + lane, im = i / (K / 8), kc = i % (K / 8);
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %4, 0;\n\t"
                     "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}"
                     ::"r"(tc::smem_u32(slot + im * HALF + kc * ROW)),
                     "l"(img + ((size_t)im * (K / 8) + kc) * NIMG + nb * CBN), "r"(ROW), "r"(tc::smem_u32(bar)),
                     "r"((int)(issuer && i < 2 * (K / 8)))
                     : "memory");
    }
}

// Column sums of one score block over the 16 rows (neighbours) of the warp's point, reduce-scattered over the 8 lanes
// that share lane % 4 (lane bits 4, 3, 2).  a[i], b[i] hold column 8 (i / 2) + 2 (lane % 4) + i % 2 of the block;
// afterwards a[0 .. CNT), b[0 .. CNT) hold columns i = base + k (same mapping) summed over all 16 rows, with
// CNT = max(CNT0 / 8, 1).  Trip counts are template parameters so that a and b stay in registers.
template <int CNT, int BIT>
__device__ __forceinline__ void ltc_reduce_scatter(float* a, float* b, int lane, int& base) {
    if constexpr (BIT >= 4) {
        if constexpr (CNT > 1) {
            constexpr int h = CNT / 2;
            const bool up = (lane & BIT) != 0;
#pragma unroll
            for (int i = 0; i < h; ++i) {
                const float ra = __shfl_xor_sync(0xffffffffu, up ? a[i] : a[i + h], BIT);
                const float rb = __shfl_xor_sync(0xffffffffu, up ? b[i] : b[i + h], BIT);
                a[i] = (up ? a[i + h] : a[i]) + ra;
                b[i] = (up ? b[i + h] : b[i]) + rb;
            }
            base += up ? h : 0;
            ltc_reduce_scatter<h, BIT / 2>(a, b, lane, base);
        } else {
            a[0] += __shfl_xor_sync(0xffffffffu, a[0], BIT);
            b[0] += __shfl_xor_sync(0xffffffffu, b[0], BIT);
            ltc_reduce_scatter<1, BIT / 2>(a, b, lane, base);
        }
    }
}

template <int D, int STAGE>
__global__ void __launch_bounds__(LtcCfg<D, STAGE>::NTH, LtcCfg<D, STAGE>::MIN_CTAS)
lfa_pool_tc_kernel(const __grid_constant__ LfaTcParams p) {
    using C = LtcCfg<D, STAGE>;
    constexpr int H = C::H, NTH = C::NTH, NPART = C::NPART, CB = C::CB, CB2 = C::CB2;
    extern __shared__ __align__(128) uint8_t smem[];
    // A buffer i: hi at smem + 2 i A_BYTES, lo right behind it
    uint8_t* b_sm = smem + C::NBUF * 2 * C::A_BYTES;  // [hi | lo] resident score weight, or two ring slots [hi | lo] each
    uint8_t* b2_sm = b_sm + 2 * C::B_BYTES;                           // [hi | lo] lse2 weight (or one column block)
    float* W10 = reinterpret_cast<float*>(b2_sm + 2 * C::B2_BYTES);  // [12][H]
    float* ST2 = W10 + 12 * H;                                       // [2][H] (+ Wl2^T [H][H] for H < 16)
    uint64_t* ring_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(W10) + C::W10_BYTES + C::ST2_BYTES);

    const int tid = threadIdx.x, lane = tid & 31;
    const int row = tid & (LTC_ROWS - 1);   // neighbour row of the tile this thread works on
    const int half = tid >> 7;              // which part of the channels / columns (0 .. NPART-1)
    // accumulator fragment of this thread (tc.cuh): rows r0 and r0 + 8 of the tile, i.e. neighbours g and g + 8 of point
    // wg * 4 + warp of the tile
    const int wg = tid >> 7, g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + ((tid >> 5) & 3) * 16 + g;
    const int pt = r0 >> 4;

    // ---- once per CTA: resident weights and the small per-channel constants
    if (!C::STREAM) {
        for (int i = tid; i < 2 * C::B_BYTES / 16; i += NTH)
            reinterpret_cast<uint4*>(b_sm)[i] = p.ws_img[i];
        if (C::MMA2)
            for (int i = tid; i < 2 * C::B2_BYTES / 16; i += NTH)
                reinterpret_cast<uint4*>(b2_sm)[i] = p.wl2_img[i];
    }
    if (STAGE == 2) {
        for (int i = tid; i < H; i += NTH) {
            ST2[i] = p.s2[i];
            ST2[H + i] = p.t2[i];
        }
        if (H < 16)
            for (int i = tid; i < H * H; i += NTH) ST2[2 * H + i] = p.wl2t[i];
    }
    for (int i = tid; i < 10 * H; i += NTH) W10[i] = p.w10t[i];
    for (int i = tid; i < H; i += NTH) {
        W10[10 * H + i] = p.s10[i];
        W10[11 * H + i] = p.t10[i];
    }
    // streamed score weight: a ring of two column blocks, filled by bulk copies.  The ring runs over the block sequence
    // 0 .. NBLK-1 of every tile in turn, so blocks 0 and 1 of the next tile are in flight during this tile's last blocks.
    uint32_t ring_phase = 0;                // bit s: parity of the next completion of slot s
    if (C::STREAM && tid == 0) {
        tc::mbar_init(&ring_full[0], 1);
        tc::mbar_init(&ring_full[1], 1);
        tc::fence_mbar_init();
    }
    tc::fence_async_smem();
    __syncthreads();
    if (C::STREAM) {
        ltc_fill<CB, D, D>(b_sm, &ring_full[0], p.ws_img, 0, lane, tid < 32);
        ltc_fill<CB, D, D>(b_sm + 2 * C::SLOT_BYTES, &ring_full[1], p.ws_img, 1, lane, tid < 32);
    }

    // The gathers are software-pipelined over tiles (d >= 64): the neighbour index of tile t+2 and the
    // coordinates / feature rows of tile t+1 are requested while tile t is worked on and land behind its
    // MMAs and epilogue (two dependent global round trips leave the per-tile critical path).  d = 256 holds 64
    // feature registers per tile: there the requests for tile t+1 go out after the rows of tile t have been stored
    // (LATE) and the index stays a raw loaded word until its tile comes up (RAW_INDEX, common.cuh RawIndex).  The
    // resident-weight kernels resolve the index of tile t+2 right behind its load.
    constexpr bool PREF = D >= 64;
    constexpr bool LATE = C::STREAM;
    constexpr bool RAW_INDEX = C::STREAM;
    constexpr int FCH = PREF ? (H / 8) / NPART : 1;      // feature chunks (8 channels) per thread
    int64_t g_nx = p.total, nb_nx = -1, g_n2 = p.total, base_n2 = -1;
    RawIndex raw_n2 = {0, 0};
    float qc_nx[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float4 f_nx[FCH][2];
    auto load_idx = [&](int64_t t, int64_t& g_, int64_t& base_, RawIndex& raw_) {
        g_ = p.total;
        base_ = -1;
        if (t < p.num_tiles) {
            g_ = t * (LTC_ROWS / LTC_K) + (row >> 4);
            if (g_ < p.total) {
                base_ = (g_ / p.n_per_batch) * p.n_per_batch;
                if (RAW_INDEX) load_index_raw(p.nidx, g_ * LTC_K + (row & 15), p.nidx_is64, raw_);
                else base_ += load_index(p.nidx, g_ * LTC_K + (row & 15), p.nidx_is64);
            }
        }
    };
    auto resolve = [&](int64_t base_, const RawIndex& raw_) -> int64_t {
        if (!RAW_INDEX) return base_;
        return base_ >= 0 ? base_ + index_value(raw_, p.nidx_is64) : (int64_t)-1;
    };
    auto load_data = [&](int64_t g_, int64_t nb_, float* qc, float4 (*f)[2]) {
        if (nb_ >= 0) {
            qc[0] = p.coords[3 * g_]; qc[1] = p.coords[3 * g_ + 1]; qc[2] = p.coords[3 * g_ + 2];
            qc[3] = p.coords[3 * nb_]; qc[4] = p.coords[3 * nb_ + 1]; qc[5] = p.coords[3 * nb_ + 2];
#pragma unroll
            for (int i = 0; i < FCH; ++i) {
                const float* src = p.feat + (size_t)nb_ * H + (half + i * NPART) * 8;
                f[i][0] = *reinterpret_cast<const float4*>(src);
                f[i][1] = *reinterpret_cast<const float4*>(src + 4);
            }
        } else {
#pragma unroll
            for (int i = 0; i < 6; ++i) qc[i] = 0.f;
#pragma unroll
            for (int i = 0; i < FCH; ++i) f[i][0] = f[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    // requests for the tile after `tile` (index resolved now, one tile after its load) and the index of the one after
    auto advance = [&](int64_t tile) {
        g_nx = g_n2;
        nb_nx = resolve(base_n2, raw_n2);
        load_data(g_nx, nb_nx, qc_nx, f_nx);
        load_idx(tile + 2 * (int64_t)gridDim.x, g_n2, base_n2, raw_n2);
    };
    if (PREF) {
        load_idx(blockIdx.x, g_nx, base_n2, raw_n2);
        nb_nx = resolve(base_n2, raw_n2);
        load_data(g_nx, nb_nx, qc_nx, f_nx);
        load_idx((int64_t)blockIdx.x + gridDim.x, g_n2, base_n2, raw_n2);
    }

    // 10-channel relative position encoding of this thread's row (randlanet.py:586-600)
    auto encode = [&](int64_t nb_, const float* qc, float* e) {
#pragma unroll
        for (int q = 0; q < 10; ++q) e[q] = 0.f;
        if (nb_ >= 0) {
            const float dx = qc[0] - qc[3], dy = qc[1] - qc[4], dz = qc[2] - qc[5];
            e[0] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            e[1] = dx; e[2] = dy; e[3] = dz;
            e[4] = qc[0]; e[5] = qc[1]; e[6] = qc[2];
            e[7] = qc[3]; e[8] = qc[4]; e[9] = qc[5];
        }
    };
    // r1 = lrelu(BN(W10 . enc)), 8 outputs at a time, straight into an operand region of H channels (chunk-major,
    // chunk `ch` of the region at dst + ch * LTC_ROWS * 16):
    //   stage 1            -> channels [H, D) of A
    //   stage 2, tensor    -> channels [0, H) of A, the A operand of the lse2 GEMM
    //   stage 2, H < 16    -> r2 = lrelu(BN(Wl2 . r1)) in registers -> channels [H, D)
    auto locse = [&](const float* e, uint8_t* dst_hi, uint8_t* dst_lo) {
        for (int ch = half; ch < H / 8; ch += NPART) {
            float r[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] = 0.f;
#pragma unroll
            for (int q = 0; q < 10; ++q) {   // warp-uniform LDS.128 of the weights
                const float4 wa = *reinterpret_cast<const float4*>(&W10[q * H + ch * 8]);
                const float4 wb = *reinterpret_cast<const float4*>(&W10[q * H + ch * 8 + 4]);
                ffma2(r[0], r[1], e[q], wa.x, wa.y);
                ffma2(r[2], r[3], e[q], wa.z, wa.w);
                ffma2(r[4], r[5], e[q], wb.x, wb.y);
                ffma2(r[6], r[7], e[q], wb.z, wb.w);
            }
            {   // folded BN + LeakyReLU; scale / shift as four LDS.128
                const float4 sa = *reinterpret_cast<const float4*>(&W10[10 * H + ch * 8]);
                const float4 sb = *reinterpret_cast<const float4*>(&W10[10 * H + ch * 8 + 4]);
                const float4 ta = *reinterpret_cast<const float4*>(&W10[11 * H + ch * 8]);
                const float4 tb = *reinterpret_cast<const float4*>(&W10[11 * H + ch * 8 + 4]);
                const float sc[8] = {sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w};
                const float sh[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float a = fmaf(r[j], sc[j], sh[j]);
                    r[j] = a >= 0.f ? a : 0.2f * a;
                }
            }
            if (STAGE == 2 && !C::MMA2) {  // H == 8: one chunk holds all of r1
                float r2[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float a = 0.f;
#pragma unroll
                    for (int i = 0; i < 8; ++i) a = fmaf(r[i], ST2[2 * H + i * H + j], a);
                    a = fmaf(a, ST2[j], ST2[H + j]);
                    r2[j] = a >= 0.f ? a : 0.2f * a;
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) r[j] = r2[j];
            }
            uint4 hi, lo;
            tc::split8(r, hi, lo);
            *reinterpret_cast<uint4*>(dst_hi + tc::op_off(LTC_ROWS, row, ch)) = hi;
            *reinterpret_cast<uint4*>(dst_lo + tc::op_off(LTC_ROWS, row, ch)) = lo;
        }
    };
    // r1 goes to channels [0, H) when the tensor core computes lse2 from it, else (r1 of stage 1, r2 of the d = 16
    // register path) to channels [H, D)
    constexpr uint32_t R1_OFF = (STAGE == 2 && C::MMA2) ? 0u : (uint32_t)(H / 8) * LTC_ROWS * 16;

    // Builds the A tile of `tile` (tiles in the CTA's order) into (a_hi, a_lo); ends with the writes fenced for the
    // tensor core, not with a barrier.  A tile past the end is built from zeros and never used.
    auto build = [&](int64_t tile, uint8_t* a_hi, uint8_t* a_lo) {
        // ---------------- neighbour id + encoding + LocSE MLP of this thread's row
        int64_t g = tile * (LTC_ROWS / LTC_K) + (row >> 4);
        int64_t nb = -1;
        float4 f_cur[FCH][2];
        if (PREF) {
            g = g_nx;
            nb = nb_nx;
            float qc[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) qc[i] = qc_nx[i];
#pragma unroll
            for (int i = 0; i < FCH; ++i) { f_cur[i][0] = f_nx[i][0]; f_cur[i][1] = f_nx[i][1]; }
            if (!LATE) advance(tile);        // tile t+1: data in flight from here; tile t+2: index
            float e[10];
            encode(nb, qc, e);
            locse(e, a_hi + R1_OFF, a_lo + R1_OFF);
        } else {
            float qc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (g < p.total) {
                const int64_t b = g / p.n_per_batch;
                nb = b * p.n_per_batch + load_index(p.nidx, g * LTC_K + (row & 15), p.nidx_is64);
                qc[0] = p.coords[3 * g]; qc[1] = p.coords[3 * g + 1]; qc[2] = p.coords[3 * g + 2];
                qc[3] = p.coords[3 * nb]; qc[4] = p.coords[3 * nb + 1]; qc[5] = p.coords[3 * nb + 2];
            }
            float e[10];
            encode(nb, qc, e);
            locse(e, a_hi + R1_OFF, a_lo + R1_OFF);
        }
        // gathered neighbour features -> channels [0, H) of A
        auto store_features = [&]() {
#pragma unroll
            for (int fi = 0; fi < (H / 8 + NPART - 1) / NPART; ++fi) {   // compile-time trip count: f_cur stays in registers
                const int ch = half + fi * NPART;
                if (ch >= H / 8) break;
                float x[8];
                if (PREF) {
                    const float4 v0 = f_cur[fi < FCH ? fi : 0][0], v1 = f_cur[fi < FCH ? fi : 0][1];
                    x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w;
                    x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
                } else if (nb >= 0) {
                    const float4 v0 = *reinterpret_cast<const float4*>(p.feat + (size_t)nb * H + ch * 8);
                    const float4 v1 = *reinterpret_cast<const float4*>(p.feat + (size_t)nb * H + ch * 8 + 4);
                    x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w;
                    x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) x[j] = 0.f;
                }
                uint4 hi, lo;
                tc::split8(x, hi, lo);
                *reinterpret_cast<uint4*>(a_hi + tc::op_off(LTC_ROWS, row, ch)) = hi;
                *reinterpret_cast<uint4*>(a_lo + tc::op_off(LTC_ROWS, row, ch)) = lo;
            }
        };

        // ---------------- stage 2: r2 = lrelu(BN(Wl2 . r1)) on the tensor core -> channels [H, D)
        if (C::MMA2) {
            tc::fence_async_smem();
            __syncthreads();
#pragma unroll 1
            for (int blk = 0; blk < H / CB2; ++blk) {
                if (C::STREAM) {   // one column block at a time through b2_sm
                    if (blk > 0) __syncthreads();    // both warpgroups' MMAs of the previous block are done with b2_sm
                    constexpr int N_U4 = H / 8 * CB2;
                    for (int i = tid; i < 2 * N_U4; i += NTH) {
                        const int im = i / N_U4, rem = i % N_U4, kc = rem / CB2, r = rem % CB2;
                        reinterpret_cast<uint4*>(b2_sm + im * C::B2_BYTES)[rem] =
                            p.wl2_img[(size_t)im * (H / 8) * H + kc * H + blk * CB2 + r];
                    }
                    tc::fence_async_smem();
                    __syncthreads();
                }
                const uint32_t bh = tc::smem_u32(b2_sm) + (C::STREAM ? 0u : (uint32_t)blk * CB2 * 16);
                float d2[CB2 / 2];
                ltc_issue<CB2, H>(d2, tc::smem_u32(a_hi), tc::smem_u32(a_lo), bh, bh + C::B2_BYTES,
                                  (C::STREAM ? CB2 : H) * 16, wg);
                ltc_wait<0, CB2 / 2>(d2);
                // r2 = lrelu(BN(.)) of the fragment, split, straight from the registers into channels [H, D) of A
#pragma unroll
                for (int q = 0; q < CB2 / 8; ++q) {
                    const int c = blk * CB2 + 8 * q + 2 * t;
                    const float2 sc = *reinterpret_cast<const float2*>(&ST2[c]);
                    const float2 sh = *reinterpret_cast<const float2*>(&ST2[H + c]);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        float v0 = fmaf(d2[4 * q + 2 * hh], sc.x, sh.x), v1 = fmaf(d2[4 * q + 2 * hh + 1], sc.y, sh.y);
                        v0 = v0 >= 0.f ? v0 : 0.2f * v0;
                        v1 = v1 >= 0.f ? v1 : 0.2f * v1;
                        const uint32_t hi = tc::cvt_f16x2(v0, v1);
                        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                        const uint32_t off = tc::op_off(LTC_ROWS, r0 + 8 * hh, (H + blk * CB2) / 8 + q) + 4 * t;
                        *reinterpret_cast<uint32_t*>(a_hi + off) = hi;
                        *reinterpret_cast<uint32_t*>(a_lo + off) = tc::cvt_f16x2(v0 - f.x, v1 - f.y);
                    }
                }
            }
            __syncthreads();   // every lse2 MMA has read r1
        }
        store_features();      // (overwrites r1 in stage 2)
        if (PREF && LATE) advance(tile);     // lands behind the score GEMM and the epilogue
        tc::fence_async_smem();
    };

    // ---------------- scores = X . Ws^T on the tensor core, CB columns per block; block j + 1 is issued before the
    // softmax over the 16 rows of the point + weighted sum of block j runs on the accumulator registers.
    // A NaN score still yields NaN: fmaxf skips it in the max, but its own exponential is NaN and enters both sums.
    auto softmax = [&](int64_t tile, const float* s, int c0, const uint8_t* a_hi, const uint8_t* a_lo) {
            const int64_t gp = tile * (LTC_ROWS / LTC_K) + pt;   // this warp's point
            constexpr int M = CB / 4;   // columns of the block in this thread's fragment
            float den[M], num[M];
#pragma unroll
            for (int q = 0; q < CB / 8; ++q) {
                // x = hi + lo of this thread's (row, column pair), rows r0 and r0 + 8
                const uint32_t off = tc::op_off(LTC_ROWS, r0, c0 / 8 + q) + 4 * t;
                const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(a_hi + off));
                const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(a_lo + off));
                const float2 h1 = __half22float2(*reinterpret_cast<const __half2*>(a_hi + off + 8 * 16));
                const float2 l1 = __half22float2(*reinterpret_cast<const __half2*>(a_lo + off + 8 * 16));
                const float x0[2] = {h0.x + l0.x, h0.y + l0.y}, x1[2] = {h1.x + l1.x, h1.y + l1.y};
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const float v0 = s[4 * q + u], v1 = s[4 * q + 2 + u];
                    float m = fmaxf(v0, v1);
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
                    const float ml = -m * kLog2e;
                    const float e0 = ex2_ftz(fmaf(v0, kLog2e, ml)), e1 = ex2_ftz(fmaf(v1, kLog2e, ml));
                    den[2 * q + u] = e0 + e1;
                    num[2 * q + u] = e0 * x0[u] + e1 * x1[u];
                }
            }
            int base = 0;
            ltc_reduce_scatter<M, 16>(den, num, lane, base);
            if (gp < p.total) {
                float* dst = p.agg + (size_t)gp * D + c0 + 8 * (base >> 1) + 2 * t;
                if (M == 16) *reinterpret_cast<float2*>(dst) = make_float2(num[0] / den[0], num[1] / den[1]);
                else if (M > 4 || !(lane & 4)) dst[base & 1] = num[0] / den[0];   // M = 4: lane bit 2 holds a copy
            }
        };
    auto issue = [&](float* d, int j, uint32_t ah, uint32_t al) {   // block j: resident weight in place, streamed weight from ring slot j % 2
            if (C::STREAM) {
                const int s = j & 1;
                tc::mbar_wait(&ring_full[s], (ring_phase >> s) & 1u);
                ring_phase ^= 1u << s;
                const uint32_t bh = tc::smem_u32(b_sm) + (uint32_t)s * 2 * C::SLOT_BYTES;
                ltc_issue<CB, D>(d, ah, al, bh, bh + C::SLOT_BYTES, CB * 16, wg);
            } else {
                const uint32_t bh = tc::smem_u32(b_sm) + (uint32_t)j * CB * 16;
                ltc_issue<CB, D>(d, ah, al, bh, bh + C::B_BYTES, D * 16, wg);
            }
        };
    float acc0[CB / 2], acc1[CB / 2];
    if (C::DBUF) {
        // tile t's two score blocks are issued, then tile t+1 is built in the other A buffer, then tile t's softmax runs
        static_assert(!C::DBUF || (C::NBLK == 2 && !C::STREAM), "double-buffered A: two resident score blocks");
        build(blockIdx.x, smem, smem + C::A_BYTES);
        __syncthreads();
        int buf = 0;
#pragma unroll 1
        for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            uint8_t* a_hi = smem + buf * 2 * C::A_BYTES;
            uint8_t* nx_hi = smem + (buf ^ 1) * 2 * C::A_BYTES;
            const uint32_t ah = tc::smem_u32(a_hi), al = ah + C::A_BYTES;
            issue(acc0, 0, ah, al);
            issue(acc1, 1, ah, al);
            build(tile + gridDim.x, nx_hi, nx_hi + C::A_BYTES);
            ltc_wait<1, CB / 2>(acc0);
            softmax(tile, acc0, 0, a_hi, a_hi + C::A_BYTES);
            ltc_wait<0, CB / 2>(acc1);
            softmax(tile, acc1, CB, a_hi, a_hi + C::A_BYTES);
            __syncthreads();   // tile t's buffer is read, tile t+1's is built
            buf ^= 1;
        }
        return;
    }
    uint8_t* a_hi = smem;
    uint8_t* a_lo = smem + C::A_BYTES;
    const uint32_t ah = tc::smem_u32(a_hi), al = tc::smem_u32(a_lo);
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        build(tile, a_hi, a_lo);
        __syncthreads();
        const bool more = tile + gridDim.x < p.num_tiles;
        auto step = [&](int j, float* cur, float* nxt) {   // block j lands in cur; block j + 1 goes to nxt
            if (j + 1 < C::NBLK) {
                issue(nxt, j + 1, ah, al);
                ltc_wait<1, CB / 2>(cur);
            } else {
                ltc_wait<0, CB / 2>(cur);
            }
            if (C::STREAM) {
                __syncthreads();      // both warpgroups are done with slot j % 2: refill it with the block two ahead
                ltc_fill<CB, D, D>(b_sm + (j & 1) * 2 * C::SLOT_BYTES, &ring_full[j & 1], p.ws_img,
                                   j + 2 < C::NBLK ? j + 2 : j + 2 - C::NBLK, lane, tid < 32 && (j + 2 < C::NBLK || more));
            }
            softmax(tile, cur, j * CB, a_hi, a_lo);
        };
        issue(acc0, 0, ah, al);
        if (C::NBLK == 1) {
            step(0, acc0, acc1);
        } else {
#pragma unroll 1
            for (int j = 0; j < C::NBLK; j += 2) {
                step(j, acc0, acc1);
                step(j + 1, acc1, acc0);
            }
        }
        __syncthreads();   // MMAs and softmax have read the A tile: free for the next tile
    }
}

template <int D, int STAGE>
static int lfa_tc_launch(const LfaTcParams& p, cudaStream_t st) {
    using C = LtcCfg<D, STAGE>;
    static_assert(C::SMEM <= 227 * 1024, "shared memory budget");
    // persistent CTAs: as many as are resident at once (registers and shared memory both limit it).  The occupancy
    // query counts the opt-in shared memory only once the kernel has been opted in.
    O3DML_CUDA(opt_in_smem<lfa_pool_tc_kernel<D, STAGE>>(C::SMEM));
    int per_sm = 0;
    O3DML_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lfa_pool_tc_kernel<D, STAGE>, C::NTH, C::SMEM));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 4) per_sm = 4;
    int64_t grid = (int64_t)device_sm_count() * per_sm;
    if (grid > p.num_tiles) grid = p.num_tiles;
    O3DML_CUDA(launch<lfa_pool_tc_kernel<D, STAGE>>((unsigned)grid, C::NTH, C::SMEM, st, p));
    return O3DML_OK;
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_randla_lfa_pool_tc(int stage, int d, const float* coords, const void* neighbor_idx,
                                        int idx_is64, int num_neighbors, const float* feat, int64_t batch,
                                        int64_t n_per_batch, const float* w10_t, const float* s10,
                                        const float* t10, const void* wl2_image, const float* wl2_t,
                                        const float* s2, const float* t2, const void* wscore_image,
                                        float* agg, void* stream) {
    O3DML_CHECK(stage == 1 || stage == 2, "lfa_tc: stage must be 1 or 2");
    O3DML_CHECK(num_neighbors == LTC_K, "lfa_tc: built for 16 neighbours");
    O3DML_CHECK(batch * n_per_batch < ((int64_t)1 << 31), "lfa_tc: too many points");
    O3DML_CHECK(stage == 1 || (s2 && t2 && (d == 16 ? wl2_t != nullptr : wl2_image != nullptr)),
                "lfa_tc: stage 2 needs the lse2 weights");
    LfaTcParams p;
    p.coords = coords; p.nidx = neighbor_idx; p.nidx_is64 = idx_is64; p.feat = feat;
    p.total = batch * n_per_batch; p.n_per_batch = n_per_batch;
    p.w10t = w10_t; p.s10 = s10; p.t10 = t10;
    p.wl2_img = (const uint4*)wl2_image; p.wl2t = wl2_t; p.s2 = s2; p.t2 = t2;
    p.ws_img = (const uint4*)wscore_image; p.agg = agg;
    p.num_tiles = ceil_div<int64_t>(p.total, LTC_ROWS / LTC_K);
    if (p.total == 0) return O3DML_OK;
    cudaStream_t st = (cudaStream_t)stream;
#define LTC_CASE(DD) \
    case DD: return stage == 1 ? lfa_tc_launch<DD, 1>(p, st) : lfa_tc_launch<DD, 2>(p, st);
    switch (d) {
        LTC_CASE(16)
        LTC_CASE(32)
        LTC_CASE(64)
        LTC_CASE(128)
        LTC_CASE(256)
        default:
            O3DML_FAIL(O3DML_ERR_UNSUPPORTED, "lfa_tc: d_out %d not in {16,32,64,128,256}", d);
    }
#undef LTC_CASE
}
