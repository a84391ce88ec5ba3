// lfa_tc.cu -- RandLA-Net attentive-pooling stage on the Hopper tensor cores (wgmma):
//   neighbour gather -> LocSE encoding (+ shared MLPs) -> score GEMM on the tensor cores with the
//   3xFP16 split (tc.cuh) -> softmax over the 16 neighbours -> weighted sum  ==> agg [N, d]
// Same contract as lfa_pool_kernel (lfa.cu); replaces randlanet.py:521-639 as used at :667-692.
//
// One tile = 128 neighbour rows = 8 points x 16 neighbours, 256 threads = two warpgroups of 64 rows (4 points each).
//   X  [128 x d]  : [feat[nbr] | r1 or r2], built by the CTA in shared memory directly in the chunk-major layout (one
//                   conflict-free 16-byte store per (row, 8 channels)), as fp16 hi/lo pairs.  In stage 2 the first
//                   half of X first holds r1 (the A operand of the lse2 GEMM) and is then overwritten by the gathered
//                   features.
//   Ws [d x d]    : score weight, host-packed hi/lo operand image [d/8][d][8]; resident in shared memory for d <= 128
//                   (d = 16, 32: zero rows up to 64), streamed for d = 256 through a ring of four 64-row x 64-k chunks
//                   filled by bulk copies (mbarrier completion), one slab's chunks after the other's
// The score product is computed channel-major, S^T = Ws . X^T: warpgroup w multiplies each 64-row slab s of Ws (the A
// operand) by its 64 rows of X (the B operand) into a [64 channels x 64 neighbour rows] accumulator (m64n64k16);
// slab s + 1 is issued into a second accumulator set before the epilogue of slab s runs.
// Epilogue on the accumulator registers: a thread holds channels g and g + 8 of the warp's 16 and, for each of the
// warpgroup's 4 points, neighbours 8q + 2t + {0, 1} (q = 0, 1): a point's 16 neighbours are 4 registers x the 4 lanes of
// a quad.  Max and the sums of e and e.x over them: the 4 registers, then lane bits 0 and 1 (max: butterfly; sums:
// reduce-scatter, after which lane t holds point t).  x = hi + lo comes from X by ldmatrix.trans, whose fragment
// (channel g, neighbours 2t, 2t + 1) is the accumulator's.
// Stage 2 chains a second GEMM (r2 = lrelu(BN(Wl2 . r1)), N = d/2) in the row-major orientation, whose epilogue writes r2
// from the registers into X (d = 16: that 8x8 product stays in registers).  The score bias is not applied: it is
// constant over the neighbours of a point and cancels in the softmax.  CTAs are persistent over tiles.  Two tiles are in
// flight per SM at d = 64 (two CTAs).
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
    static constexpr int NS = D < 64 ? 1 : D / 64;   // score-channel slabs of 64 weight rows
    static constexpr int WROWS = NS * 64;            // rows of the weight in shared memory (d < 64: zero rows up to 64)
    // streamed weight: a slab in chunks of 64 k, one ring slot each (hi, then lo); the ring holds one slab
    static constexpr int KCH = 64;
    static constexpr int NKC = STREAM ? D / KCH : 1;
    static constexpr int CHUNK_HALF = KCH / 8 * 64 * 16;
    static constexpr int CB2 = STREAM ? 32 : (H < 64 ? H : 64);  // lse2 columns per block
    static constexpr int A_BYTES = D / 8 * LTC_ROWS * 16;  // one of hi / lo
    static constexpr int W_HALF = STREAM ? CHUNK_HALF : D / 8 * WROWS * 16;  // lo behind hi (resident image, ring slot)
    static constexpr int W_BYTES = NKC * 2 * W_HALF;
    static constexpr int B2_BYTES = MMA2 ? (STREAM ? H / 8 * CB2 * 16 : H / 8 * H * 16) : 0;
    static constexpr int W10_BYTES = 12 * H * 4;
    static constexpr int ST2_BYTES = STAGE == 2 ? (2 * H + (H < 16 ? H * H : 0)) * 4 : 0;
    // Two tiles in flight per SM at d = 64, as two CTAs (<= 128 registers), so that the SIMT build of one tile overlaps
    // the score MMAs of the other.  d = 128 and 256 have room for one.
    static constexpr int MIN_CTAS = D == 64 ? 2 : 1;
    static constexpr size_t SMEM = 2 * A_BYTES + W_BYTES + 2 * B2_BYTES + W10_BYTES + ST2_BYTES + 8 * NKC + 128;
};

// Issues (does not wait for) D[64 x N] (+)= A[64 x K] . B[N x K]^T -> d[N / 2] as one committed wgmma group.  Each
// operand is a hi / lo pair of chunk-major images addressed at its first row (rows 16 bytes apart, 8-k chunks lbo
// apart); the three products of the split run in the order hi.hi, hi.lo, lo.hi.  With `acc` the group adds to d.  SET
// overwrites d without reading it: its old values need not be live (the score accumulators, two sets of 32 registers,
// would otherwise stay live across the tile build).
template <int N, int K, bool SET = false>
__device__ __forceinline__ void ltc_issue(float* d, uint32_t a_hi, uint32_t a_lo, uint32_t a_lbo, uint32_t b_hi,
                                          uint32_t b_lo, uint32_t b_lbo, bool acc) {
    if (!SET) {
#pragma unroll
        for (int i = 0; i < N / 2; ++i) tc::fence_operand(d[i]);
    }
    tc::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < K / 16; ++ks) {
        const uint64_t ah = tc::smem_desc(a_hi + ks * 2 * a_lbo, a_lbo, 128);
        const uint64_t al = tc::smem_desc(a_lo + ks * 2 * a_lbo, a_lbo, 128);
        const uint64_t bh = tc::smem_desc(b_hi + ks * 2 * b_lbo, b_lbo, 128);
        const uint64_t bl = tc::smem_desc(b_lo + ks * 2 * b_lbo, b_lbo, 128);
        if constexpr (SET) {
            if (ks == 0) tc::wgmma_f16_ss_set<N>(d, ah, bh);
            else tc::wgmma_f16_ss<N>(d, ah, bh, 1u);
        } else {
            tc::wgmma_f16_ss<N>(d, ah, bh, acc || ks > 0);
        }
        tc::wgmma_f16_ss<N>(d, ah, bl, 1u);
        tc::wgmma_f16_ss<N>(d, al, bh, 1u);
    }
    tc::wgmma_commit();
#pragma unroll
    for (int i = 0; i < N / 2; ++i) tc::fence_operand(d[i]);
}

// Waits until at most N of this warpgroup's wgmma groups are pending; d (the oldest group's accumulators) is then final
template <int N, int CNT>
__device__ __forceinline__ void ltc_wait(float* d) {
    tc::wgmma_wait<N>();
#pragma unroll
    for (int i = 0; i < CNT; ++i) tc::fence_operand(d[i]);
}

// One bulk copy (TMA) per (hi / lo, 8-k chunk) of chunk kc (k in [KCH kc, KCH kc + KCH)) of the 64 rows of slab s of
// the score weight image [D/8][D][8] (hi, then lo) into a ring slot [hi | lo] of [KCH/8][64][8] each, completing on
// bar.  Every thread of the CTA runs it and the lanes of the warp with `issuer` set issue the copies: the instructions
// are predicated rather than branched around, because a divergent branch while a wgmma group is in flight makes ptxas
// serialize the wgmma instructions.
template <int D, int KCH>
__device__ __forceinline__ void ltc_fill(uint8_t* slot, uint64_t* bar, const uint4* __restrict__ img, int s, int kc,
                                         int lane, bool issuer) {
    constexpr uint32_t ROW = 64 * 16, HALF = KCH / 8 * ROW;
    constexpr int NCP = 2 * (KCH / 8);
    static_assert(NCP <= 32, "one copy per lane");
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t"
                 "@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(tc::smem_u32(bar)),
                 "r"(2 * HALF), "r"((int)(issuer && lane == 0))
                 : "memory");
    const int im = lane / (KCH / 8), k8 = lane % (KCH / 8);
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %4, 0;\n\t"
                 "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}"
                 ::"r"(tc::smem_u32(slot + (im & 1) * HALF + k8 * ROW)),
                 "l"(img + ((size_t)(im & 1) * (D / 8) + kc * (KCH / 8) + k8) * D + s * 64), "r"(ROW),
                 "r"(tc::smem_u32(bar)), "r"((int)(issuer && lane < NCP))
                 : "memory");
}

// With NKC wgmma groups pending, runs f(kc) for kc = KC .. NKC - 1, each as soon as group kc has completed
// (wait_group NKC - 1 - kc)
template <int KC, int NKC, class F>
__device__ __forceinline__ void ltc_release(F&& f) {
    if constexpr (KC < NKC) {
        tc::wgmma_wait<NKC - 1 - KC>();
        f(KC);
        ltc_release<KC + 1, NKC>(f);
    }
}

// Sums over the 4 lanes of a quad (lane bits 1, 0; call with BIT = 2) as a reduce-scatter: a[i], b[i] hold this lane's
// partial of pair i; afterwards a[0 .. CNT), b[0 .. CNT) hold pairs base + k summed over the quad, with
// CNT = CNT0 / 4 (CNT0 >= 4).  Each pair's sum is (v0 + v2) + (v1 + v3) of the lanes' partials, whichever lane ends up
// with it.  Trip counts are template parameters so that a and b stay in registers.
template <int CNT, int BIT>
__device__ __forceinline__ void ltc_reduce_scatter(float* a, float* b, int lane, int& base) {
    if constexpr (BIT >= 1) {
        static_assert(CNT > 1, "one pair per lane and bit at least");
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
    }
}

template <int D, int STAGE>
__global__ void __launch_bounds__(LtcCfg<D, STAGE>::NTH, LtcCfg<D, STAGE>::MIN_CTAS)
lfa_pool_tc_kernel(const __grid_constant__ LfaTcParams p) {
    using C = LtcCfg<D, STAGE>;
    constexpr int H = C::H, NTH = C::NTH, NPART = C::NPART, NS = C::NS, NKC = C::NKC, CB2 = C::CB2;
    extern __shared__ __align__(128) uint8_t smem[];
    // X tile: hi at smem, lo right behind it
    uint8_t* w_sm = smem + 2 * C::A_BYTES;  // [hi | lo] resident score weight, or NKC ring slots [hi | lo] each
    uint8_t* b2_sm = w_sm + C::W_BYTES;                               // [hi | lo] lse2 weight (or one column block)
    float* W10 = reinterpret_cast<float*>(b2_sm + 2 * C::B2_BYTES);  // [12][H]
    float* ST2 = W10 + 12 * H;                                       // [2][H] (+ Wl2^T [H][H] for H < 16)
    uint64_t* ring_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(W10) + C::W10_BYTES + C::ST2_BYTES);

    const int tid = threadIdx.x, lane = tid & 31;
    const int row = tid & (LTC_ROWS - 1);   // neighbour row of the tile this thread works on
    const int half = tid >> 7;              // which part of the channels / columns (0 .. NPART-1)
    // accumulator fragment of this thread in the lse2 product (tc.cuh): rows r0 and r0 + 8 of the tile
    const int wg = tid >> 7, g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + ((tid >> 5) & 3) * 16 + g;

    // ---- once per CTA: resident weights and the small per-channel constants
    if (!C::STREAM) {
        // [hi | lo][D/8][WROWS][8] from the image [hi | lo][D/8][D][8]; rows past d (d < 64) are zero
        for (int i = tid; i < C::W_BYTES / 16; i += NTH) {
            const int r = i % C::WROWS, kc = i / C::WROWS;
            reinterpret_cast<uint4*>(w_sm)[i] = r < D ? p.ws_img[kc * D + r] : make_uint4(0u, 0u, 0u, 0u);
        }
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
    // streamed score weight: slot kc of the ring holds chunk kc of a slab.  The ring runs over the slabs 0 .. NS-1 of
    // every tile in turn, all slots completing once per slab, so one parity serves them all; slab 0 of the next tile
    // arrives while this tile's last slab is worked on.
    uint32_t ring_phase = 0;
    if (C::STREAM && tid == 0) {
        for (int kc = 0; kc < NKC; ++kc) tc::mbar_init(&ring_full[kc], 1);
        tc::fence_mbar_init();
    }
    tc::fence_async_smem();
    __syncthreads();
    if (C::STREAM) {
#pragma unroll
        for (int kc = 0; kc < NKC; ++kc)
            ltc_fill<D, C::KCH>(w_sm + kc * 2 * C::W_HALF, &ring_full[kc], p.ws_img, 0, kc, lane, tid < 32);
    }

    // The gathers are software-pipelined over tiles (d >= 64): the neighbour index of tile t+2 and the
    // coordinates / feature rows of tile t+1 are requested while tile t is worked on and land behind its
    // MMAs and epilogue (two dependent global round trips leave the per-tile critical path).  d = 256 holds 64
    // feature registers per tile, which do not fit next to the two 32-register score accumulator sets: there the
    // requests for tile t+1 go out once the last score slab's MMAs are done, behind its softmax (LATE), and the index
    // stays a raw loaded word until its tile comes up (RAW_INDEX, common.cuh RawIndex).  The
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
                ltc_issue<CB2, H>(d2, tc::smem_u32(a_hi) + wg * 64 * 16, tc::smem_u32(a_lo) + wg * 64 * 16,
                                  LTC_ROWS * 16, bh, bh + C::B2_BYTES, (C::STREAM ? CB2 : H) * 16, false);
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
        tc::fence_async_smem();
    };

    // ---------------- scores S^T = Ws . X^T on the tensor core, one 64-channel slab at a time; slab j + 1 is issued
    // before the softmax over the 16 neighbours of each point + weighted sum of slab j runs on the accumulator registers.
    // Accumulator register 8p + 4q + 2h + u of a thread is channel 64 slab + 16 warp + 8h + g, neighbour 8q + 2t + u
    // of the warpgroup's point p (tc.cuh).
    // A NaN score still yields NaN: fmaxf skips it in the max, but its own exponential is NaN and enters both sums.
    auto softmax = [&](int64_t tile, const float* s, int slab, uint32_t x_hi, uint32_t x_lo) {
            const int c0 = slab * 64 + ((tid >> 5) & 3) * 16;   // channel of this warp's accumulator row 0
            const bool live = c0 < D;                           // d < 64: the warps past d hold zero rows of the slab
            // ldmatrix rows: lanes 8j .. 8j + 7 address matrix j = neighbour rows 32pp + 8j .. + 7 of the warpgroup
            const uint32_t x0 = (uint32_t)(live ? c0 / 8 : 0) * LTC_ROWS * 16 + (uint32_t)(wg * 64 + lane) * 16;
#pragma unroll
            for (int h = 0; h < 2; ++h) {   // channel 8h + g
                float den[4], num[4];       // point p
#pragma unroll
                for (int pp = 0; pp < 2; ++pp) {
                    // x = hi + lo at neighbours 8q + 2t, 8q + 2t + 1 of points 2pp, 2pp + 1, q = 0, 1
                    uint32_t xh[4], xl[4];
                    const uint32_t off = x0 + (uint32_t)h * LTC_ROWS * 16 + (uint32_t)pp * 32 * 16;
                    tc::ldsm_x4_trans(xh, x_hi + off);
                    tc::ldsm_x4_trans(xl, x_lo + off);
#pragma unroll
                    for (int pl = 0; pl < 2; ++pl) {
                        const int pq = 2 * pp + pl;
                        float v[4], x[4];
#pragma unroll
                        for (int q = 0; q < 2; ++q) {
                            const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&xh[2 * pl + q]));
                            const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&xl[2 * pl + q]));
                            v[2 * q] = s[8 * pq + 4 * q + 2 * h];
                            v[2 * q + 1] = s[8 * pq + 4 * q + 2 * h + 1];
                            x[2 * q] = fh.x + fl.x;
                            x[2 * q + 1] = fh.y + fl.y;
                        }
                        float m = fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3]));
                        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
                        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
                        const float ml = -m * kLog2e;
                        float e[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) e[k] = ex2_ftz(fmaf(v[k], kLog2e, ml));
                        den[pq] = (e[0] + e[1]) + (e[2] + e[3]);
                        num[pq] = fmaf(e[1], x[1], e[0] * x[0]) + fmaf(e[3], x[3], e[2] * x[2]);
                    }
                }
                int base = 0;
                ltc_reduce_scatter<4, 2>(den, num, lane, base);   // lane t: point t
                const int64_t gp = tile * (LTC_ROWS / LTC_K) + wg * 4 + base;
                if (live && gp < p.total) p.agg[(size_t)gp * D + c0 + 8 * h + g] = num[0] / den[0];
            }
        };
    // slab j against X (hi at x_hi, lo at x_lo): the resident weight in place, or the streamed one from the ring, one
    // wgmma group per chunk as soon as the chunk has landed (the last chunk's copy starts as the previous slab ends)
    auto issue = [&](float* d, int j, uint32_t x_hi, uint32_t x_lo) {
            const uint32_t bh = x_hi + wg * 64 * 16, bl = x_lo + wg * 64 * 16;
            const uint32_t w = tc::smem_u32(w_sm);
            if (C::STREAM) {
                tc::mbar_wait(&ring_full[0], ring_phase);
                ltc_issue<64, C::KCH, true>(d, w, w + C::W_HALF, 64 * 16, bh, bl, LTC_ROWS * 16, false);
#pragma unroll
                for (int kc = 1; kc < NKC; ++kc) {
                    const uint32_t a = w + kc * 2 * C::W_HALF, xo = kc * (C::KCH / 8) * LTC_ROWS * 16;
                    tc::mbar_wait(&ring_full[kc], ring_phase);
                    ltc_issue<64, C::KCH>(d, a, a + C::W_HALF, 64 * 16, bh + xo, bl + xo, LTC_ROWS * 16, true);
                }
                ring_phase ^= 1u;
            } else {
                const uint32_t a = w + j * 64 * 16;
                ltc_issue<64, D, true>(d, a, a + C::W_HALF, C::WROWS * 16, bh, bl, LTC_ROWS * 16, false);
            }
        };
    float acc0[32], acc1[32];
    uint8_t* a_hi = smem;
    uint8_t* a_lo = smem + C::A_BYTES;
    const uint32_t ah = tc::smem_u32(a_hi), al = tc::smem_u32(a_lo);
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        build(tile, a_hi, a_lo);
        __syncthreads();
        const bool more = tile + gridDim.x < p.num_tiles;
        auto step = [&](int j, float* cur, float* nxt) {   // slab j lands in cur; slab j + 1 goes to nxt
            if (C::STREAM) {
                // as each chunk group of slab j completes, both warpgroups are done with its slot: refill it with the
                // same chunk of the next slab (slab 0 of the next tile after the last)
                ltc_release<0, NKC>([&](int kc) {
                    __syncthreads();
                    ltc_fill<D, C::KCH>(w_sm + kc * 2 * C::W_HALF, &ring_full[kc], p.ws_img, j + 1 < NS ? j + 1 : 0,
                                        kc, lane, tid < 32 && (j + 1 < NS || more));
                });
#pragma unroll
                for (int i = 0; i < 32; ++i) tc::fence_operand(cur[i]);
                if (j + 1 < NS) issue(nxt, j + 1, ah, al);
                else if (PREF && LATE) advance(tile);   // lands behind the last softmax
            } else if (j + 1 < NS) {
                issue(nxt, j + 1, ah, al);
                ltc_wait<1, 32>(cur);
            } else {
                ltc_wait<0, 32>(cur);
            }
            softmax(tile, cur, j, ah, al);
        };
        issue(acc0, 0, ah, al);
        if (NS == 1) {
            step(0, acc0, acc1);
        } else {
#pragma unroll   // unrolled: no wgmma group is in flight across a back-edge, which ptxas would serialize
            for (int j = 0; j < NS; j += 2) {
                step(j, acc0, acc1);
                step(j + 1, acc1, acc0);
            }
        }
        __syncthreads();   // MMAs and softmax have read the X tile: free for the next tile
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
