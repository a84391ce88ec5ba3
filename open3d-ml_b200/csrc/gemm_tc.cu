// gemm_tc.cu -- the gathered GEMM / implicit-GEMM convolution of gemm.cu on the Hopper tensor cores (wgmma):
// 3xTF32 split, operands staged by the TMA engine.
//
//   D[128 x BN] = A[128 x K] * W[K x BN], fp32 in / fp32 out, accumulated in registers.
//
// Precision.  TF32 keeps fp32's exponent, so no range pass, no power-of-two scaling and no clamp are
// needed.  x = hi + lo with hi = x & 0xFFFFE000 (the 10 explicit mantissa bits TF32 keeps) and lo = x - hi
// (exact in fp32, <= 13 bits of which the tensor core keeps 11): A*W ~= Ah*Wh + Ah*Wl + Al*Wh, relative
// error ~2^-21 per product (tests/test_split_numerics.py emulates it on the CPU).
// The weight side is split by the host (round-to-nearest, _lib.pack_linear).
//
// Data movement.  The raw fp32 A slice (128 rows x 32 channels = 128 B per row) IS the hi operand:
//   * identity row sources and the 3x3 convolution taps are fetched by ONE cp.async.bulk.tensor per
//     slice (2-D {channels, rows} map; 4-D {C, W, H, B} map whose box is a PW x PH patch of output
//     pixels shifted by the tap -- negative / overflowing coordinates are zero-filled by the TMA unit,
//     which is the convolution padding; stride-2 convolutions use four parity maps),
//   * gathered sources (index / batch-relative index / shadow rows) by 16-byte cp.async into the same
//     128-byte-swizzled layout,
//   * the weight slices (hi and lo image) by two more tensor copies.
// The two consumer warpgroups (64 rows each) read their A fragments straight from the swizzled tile into
// registers, split them there (hi = x & mask, lo = x - hi) and issue register-A wgmma against the W hi / lo
// tiles in shared memory: the split never goes back to shared memory.
// Shared-memory layout: K-major, SWIZZLE_128B (row r, 16-byte chunk c at r*128 + ((c ^ (r & 7)) << 4)),
// descriptors with SBO = 1024, K advanced by +32 B per wgmma (K = 8 TF32).
//
// Every GT_FLUSH slices the wgmma accumulator is folded into a second fp32 register set with
// round-to-nearest adds, so that long products do not rely on the tensor core's internal accumulation.
#include "../../include/o3dml_b200.h"
#include "dense.cuh"
#include "tc.cuh"
#include <cuda.h>
#include <algorithm>

namespace o3dml {

constexpr int GT_ROWS = 128;
constexpr int GT_KS = 32;        // fp32 channels per k-slice (= one 128-byte swizzle row)
constexpr int GT_FLUSH = 4;      // k-slices (128 channels = 48 accumulating MMAs) per register accumulation chunk
constexpr int GT_MAX_SRC = 3;
constexpr int GT_CONV_THREADS = 256;   // warps 0-7: the two consumer warpgroups
constexpr int GT_LOADERS = 128;        // warps 8-11 (GATHER kernels only)
constexpr int GT_A_BYTES = GT_ROWS * 128;

struct alignas(64) GemmTcParams {
    CUtensorMap mapA[4];   // rows mode: one per identity source; conv: stride 1 -> [0], stride 2 -> parity (py*2+px)
    CUtensorMap mapB;      // {Kpad, 2*Npad}: hi rows [0, Npad), lo rows [Npad, 2*Npad)
    int64_t N;
    int K, Kpad, Cout, Npad;
    int mode;  // 0 rows, 1 conv3x3
    int nsrc;
    o3dml_src_t src[GT_MAX_SRC];
    int koff[GT_MAX_SRC + 1];
    int H, W, OH, OW, stride, C;
    int lpw, PH, tiles_x, tiles_y;   // conv: patch = (1 << lpw) x PH output pixels per CTA
    DenseEpilogue ep;
};

// ---- async-copy primitives ---------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes)
                 : "memory");
}
// the mbarrier gets one (pre-counted) arrival from this thread once all of its earlier cp.async have landed
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(tc::smem_u32(bar)) : "memory");
}
using tc::mbar_arrive_expect_tx;
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc::smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// TMA tiled loads (cp.async.bulk.tensor), completion counted in bytes on the mbarrier
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_dst),
        "l"(map), "r"(tc::smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(smem_dst),
        "l"(map), "r"(tc::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// LITE: two stages instead of 4 - 6, so that TWO CTAs share an SM.  A short product (K <= 512) is mostly
// prologue and epilogue around a few 32-channel slices: with one CTA per SM the tensor pipe and the TMA unit
// idle through both; a sibling CTA fills them.
template <int BN, bool LITE = false>
struct GtCfg {
    static constexpr int B_BYTES = BN * 128;                       // one of hi/lo per stage
    static constexpr int STAGE = GT_A_BYTES + 2 * B_BYTES;         // raw A + W hi + W lo; multiples of 1024
    static constexpr int STAGES = LITE ? 2 : BN >= 128 ? 4 : 6;
    static_assert(!LITE || BN <= 64, "LITE is for the narrow tiles");
    static constexpr int TAIL = GT_MAX_SRC * GT_ROWS * 8 + GT_ROWS * 8 + 2 * BN * 4 + 256;
    static constexpr size_t SMEM = (size_t)STAGES * STAGE + TAIL + 1024;
    static_assert(SMEM <= 227 * 1024, "shared memory budget of one H100 CTA");
    static_assert((size_t)STAGES * STAGE >= (size_t)GT_ROWS * (BN + 4) * 4, "epilogue staging lives in the stages");
};

// Pipeline (per CTA, one [128 x BN] output tile, k-slices of 32 channels through a ring of stages):
//   warps 0-7     two consumer warpgroups (rows 0-63, 64-127): wait full[stage], load and split the A
//                 fragments of their rows, issue 12 wgmma (4 k-steps x 3 products), wait for them, arrive
//                 empty[stage]; fold the accumulator every GT_FLUSH slices; epilogue (BN / residual /
//                 activation through shared-memory staging, row-coalesced stores)
//   warp 8 lane 0 TMA producer: waits empty[stage], arms full[stage] with the byte count and issues the
//                 weight-slice copies and -- for identity sources / convolution taps -- the A copy
//   warps 8-11    (GATHER kernels, lane 0 of warp 8 included) loaders: 16-byte cp.async of gathered rows into the
//                 swizzled A tile, cp.async.mbarrier.arrive on full[stage].  Sharing warp 8 keeps the block at 384
//                 threads: 168 registers per thread, which the 2 x BN / 2 accumulator and fold registers need at BN = 128
constexpr int GT_PRODUCER_WARP = 8;

template <bool GATHER>
__host__ __device__ constexpr int gt_threads() { return GT_CONV_THREADS + (GATHER ? GT_LOADERS : 32); }

template <int BN, bool GATHER, bool LITE>
__global__ void __launch_bounds__(gt_threads<GATHER>(), LITE ? 2 : 1)
gemm_tc_kernel(const __grid_constant__ GemmTcParams p) {
    using C = GtCfg<BN, LITE>;
    constexpr int S = C::STAGES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = tc::smem_u32(smem_raw);
    uint8_t* stages = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);           // 1024-byte aligned
    const float** rowptr = reinterpret_cast<const float**>(stages + S * C::STAGE);   // [src][row]
    int64_t* rown = reinterpret_cast<int64_t*>(rowptr + GT_MAX_SRC * GT_ROWS);       // [row] output row or -1
    float* s_scale = reinterpret_cast<float*>(rown + GT_ROWS);                       // [BN] folded BN scale of this column tile
    float* s_shift = s_scale + BN;                                                   // [BN]
    uint64_t* mbar = reinterpret_cast<uint64_t*>(s_shift + BN);
    uint64_t* full_bar = mbar;                // [S] operands of the slice landed
    uint64_t* empty_bar = mbar + S;           // [S] the consumers are done with the stage

    const DenseEpilogue& ep = p.ep;
    const int tid = threadIdx.x;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // warp-uniform for the compiler
    const int col0 = blockIdx.y * BN;
    // rows mode: 128 consecutive output rows; conv mode: a PW x PH patch of output pixels of one image
    int64_t row0 = (int64_t)blockIdx.x * GT_ROWS;
    int cb = 0, oy0 = 0, ox0 = 0;
    if (p.mode == 1) {
        const int per = p.tiles_x * p.tiles_y;
        cb = blockIdx.x / per;
        const int t = blockIdx.x - cb * per;
        oy0 = (t / p.tiles_x) * p.PH;
        ox0 = (t % p.tiles_x) << p.lpw;
    }

    // ---- per-row bookkeeping
    for (int m = tid; m < GT_ROWS; m += blockDim.x) {
        int64_t n;
        if (p.mode == 0) {
            n = row0 + m;
            if (n >= p.N) n = -1;
        } else {
            const int oy = oy0 + (m >> p.lpw), ox = ox0 + (m & ((1 << p.lpw) - 1));
            n = (oy < p.OH && ox < p.OW) ? ((int64_t)cb * p.OH + oy) * p.OW + ox : -1;
        }
        rown[m] = n;
    }
    for (int i = tid; i < BN; i += blockDim.x) {      // per-column epilogue constants: read once, not per element
        const int c = col0 + i;
        s_scale[i] = (ep.scale && c < p.Cout) ? ep.scale[c] : 1.f;
        s_shift[i] = (ep.shift && c < p.Cout) ? ep.shift[c] : 0.f;
    }
    if (GATHER) {
        for (int i = tid; i < p.nsrc * GT_ROWS; i += blockDim.x) {
            const int s = i / GT_ROWS, m = i % GT_ROWS;
            const int64_t n = row0 + m;
            rowptr[s * GT_ROWS + m] = (n < p.N && p.src[s].index) ? src_row(p.src[s], n) : nullptr;
        }
    }
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < S; ++i) {
            tc::mbar_init(&full_bar[i], GATHER ? 1 + GT_LOADERS : 1);
            tc::mbar_init(&empty_bar[i], GT_CONV_THREADS);
        }
        tc::fence_mbar_init();
    }
    __syncthreads();

    const int nsl = p.Kpad / GT_KS;
    const uint32_t stage0 = tc::smem_u32(stages);

    if (warp >= GT_PRODUCER_WARP) {
        // ================================================================= TMA producer (+ gather loaders)
        const int rt = tid - GT_CONV_THREADS;                   // loader index; 0 is also the producer
        if (GATHER || rt == 0) {
            if (rt == 0) tma_prefetch_desc(&p.mapB);
            const int spt = p.mode == 1 ? p.C / GT_KS : 1;      // slices per convolution tap
            int sidx = 0;
            for (int sl = 0; sl < nsl; ++sl) {
                const int stage = sl % S, use = sl / S;
                if (use >= 1) tc::mbar_wait(&empty_bar[stage], (use - 1) & 1);
                const int k0 = sl * GT_KS;
                bool a_tma = true;
                if (p.mode == 0) {
                    while (sidx + 1 < p.nsrc && k0 >= p.koff[sidx + 1]) ++sidx;
                    a_tma = p.src[sidx].index == nullptr;
                }
                const uint32_t ah = stage0 + (uint32_t)stage * C::STAGE;
                if (rt == 0) {
                    const uint32_t bh = ah + GT_A_BYTES;
                    mbar_arrive_expect_tx(&full_bar[stage], 2 * C::B_BYTES + (a_tma ? GT_A_BYTES : 0));
                    tma_load_2d(bh, &p.mapB, k0, col0, &full_bar[stage]);
                    tma_load_2d(bh + C::B_BYTES, &p.mapB, k0, p.Npad + col0, &full_bar[stage]);
                    if (a_tma) {
                        if (p.mode == 0) {
                            tma_load_2d(ah, &p.mapA[sidx], k0 - p.koff[sidx], (int)row0, &full_bar[stage]);
                        } else {
                            const int tap = sl / spt, cc = (sl - tap * spt) * GT_KS;
                            const int dy = tap / 3, dx = tap - dy * 3;
                            if (p.stride == 1) {
                                tma_load_4d(ah, &p.mapA[0], cc, ox0 - 1 + dx, oy0 - 1 + dy, cb, &full_bar[stage]);
                            } else {   // input pixel 2*o - 1 + d: odd parity for d = 0 (coordinate o - 1) and d = 2 (o)
                                const int py = dy != 1, px = dx != 1;
                                tma_load_4d(ah, &p.mapA[py * 2 + px], cc, ox0 - (dx == 0), oy0 - (dy == 0), cb,
                                            &full_bar[stage]);
                            }
                        }
                    }
                }
                if (!GATHER) continue;
                if (!a_tma) {
                    const int kloc = k0 - p.koff[sidx];
                    const int cs = p.src[sidx].channels;
#pragma unroll
                    for (int j = 0; j < (GT_ROWS * 8) / GT_LOADERS; ++j) {     // 8 consecutive lanes = one row's 128 B
                        const int item = rt + j * GT_LOADERS;
                        const int m = item >> 3, c = item & 7;
                        const float* base = rowptr[sidx * GT_ROWS + m];
                        const int kk = kloc + c * 4;
                        const bool ok = base != nullptr && kk < cs;
                        cp_async16(ah + (uint32_t)m * 128u + (uint32_t)((c ^ (m & 7)) << 4),
                                   ok ? (const void*)(base + kk) : (const void*)p.src[0].data, ok ? 16 : 0);
                    }
                    cp_async_arrive(&full_bar[stage]);
                } else {
                    mbar_arrive(&full_bar[stage]);
                }
            }
        }
    } else if (warp < GT_PRODUCER_WARP) {
        // ================================================================= consumers + fold + epilogue
        const int lane = tid & 31, g = lane >> 2, t = lane & 3;
        const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + g;      // fragment rows r0 and r0 + 8
        constexpr int ND = BN / 2;                                  // accumulator registers per thread
        float acc[ND], racc[ND];
#pragma unroll
        for (int i = 0; i < ND; ++i) { acc[i] = 0.f; racc[i] = 0.f; }
        for (int s = 0; s < nsl; ++s) {
            const int stage = s % S, use = s / S;
            tc::mbar_wait(&full_bar[stage], use & 1);
            // A fragments of this thread (m16n8k8 TF32: (r0, t), (r0+8, t), (r0, t+4), (r0+8, t+4) per k-step),
            // read from the swizzled tile: the 32 lanes of a warp hit 32 different banks
            const uint8_t* a_tile = stages + (size_t)stage * C::STAGE;
            uint32_t ah[GT_KS / 8][4], al[GT_KS / 8][4];
#pragma unroll
            for (int ks = 0; ks < GT_KS / 8; ++ks)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = r0 + (e & 1) * 8, k = ks * 8 + t + (e >> 1) * 4;
                    const uint32_t x = *reinterpret_cast<const uint32_t*>(
                        a_tile + r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4);
                    tc::split_tf32(x, ah[ks][e], al[ks][e]);
                }
            const uint32_t bh = stage0 + (uint32_t)stage * C::STAGE + GT_A_BYTES, bl = bh + C::B_BYTES;
            const uint32_t first = (s % GT_FLUSH) != 0;            // 0: this slice starts a new accumulation chunk
            tc::wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < GT_KS / 8; ++ks) {        // K = 8 TF32 = 32 bytes of W per wgmma
                tc::wgmma_tf32_rs<BN>(acc, ah[ks], tc::smem_desc_sw128(bh + ks * 32), ks == 0 ? first : 1u);
                tc::wgmma_tf32_rs<BN>(acc, ah[ks], tc::smem_desc_sw128(bl + ks * 32), 1u);
                tc::wgmma_tf32_rs<BN>(acc, al[ks], tc::smem_desc_sw128(bh + ks * 32), 1u);
            }
            tc::wgmma_commit();
            tc::wgmma_wait_all();
            mbar_arrive(&empty_bar[stage]);
            if ((s % GT_FLUSH) == GT_FLUSH - 1 || s == nsl - 1) {
#pragma unroll
                for (int i = 0; i < ND; ++i) racc[i] += acc[i];
            }
        }
        // ---- epilogue: the tile goes through the (now dead) pipeline stages so that the global stores are
        // whole rows (row-major / pixel shuffle) or whole pixel runs (NCHW) written by consecutive lanes
        named_bar_sync(1, GT_CONV_THREADS);                          // every consumer is done with the stages
        constexpr int SLD = BN + 4;                                  // staging row stride (floats)
        float* stg = reinterpret_cast<float*>(stages);
#pragma unroll
        for (int i = 0; i < ND; i += 2) {
            const int r = r0 + ((i >> 1) & 1) * 8, c = (i >> 2) * 8 + 2 * t;
            *reinterpret_cast<float2*>(stg + r * SLD + c) =
                make_float2(fmaf(racc[i], s_scale[c], s_shift[c]), fmaf(racc[i + 1], s_scale[c + 1], s_shift[c + 1]));
        }
        named_bar_sync(2, GT_CONV_THREADS);
        const bool staged = ep.mode == 0 || (ep.mode == 2 && (ep.dC & 3) == 0);
        if (staged) {
            constexpr int LPR = BN / 4;                                // lanes per output row
            const int c = (tid % LPR) * 4, cg = col0 + c;
            const bool vec = (ep.out_ld & 3) == 0 && (reinterpret_cast<uintptr_t>(ep.out) & 15) == 0;
            if (cg < p.Cout) {
                for (int r = tid / LPR; r < GT_ROWS; r += GT_CONV_THREADS / LPR) {
                    const int64_t nr = rown[r];
                    if (nr < 0) continue;
                    float4 v = *reinterpret_cast<const float4*>(stg + r * SLD + c);
                    if (ep.residual) {
                        const float* rp = ep.residual + (size_t)nr * ep.res_ld + cg;
                        if (cg + 3 < p.Cout && (ep.res_ld & 3) == 0 && (reinterpret_cast<uintptr_t>(ep.residual) & 15) == 0) {
                            const float4 rv = *reinterpret_cast<const float4*>(rp);
                            v.x += rv.x; v.y += rv.y; v.z += rv.z; v.w += rv.w;
                        } else {
                            if (cg < p.Cout) v.x += rp[0];
                            if (cg + 1 < p.Cout) v.y += rp[1];
                            if (cg + 2 < p.Cout) v.z += rp[2];
                            if (cg + 3 < p.Cout) v.w += rp[3];
                        }
                    }
                    v.x = apply_act(v.x, ep.act, ep.slope); v.y = apply_act(v.y, ep.act, ep.slope);
                    v.z = apply_act(v.z, ep.act, ep.slope); v.w = apply_act(v.w, ep.act, ep.slope);
                    float* o;
                    if (ep.mode == 0) {
                        o = ep.out + (size_t)nr * ep.out_ld + cg;
                    } else {
                        const int64_t per = (int64_t)ep.dIH * ep.dIW;
                        const int64_t b = nr / per;
                        const int rr = (int)(nr % per);
                        const int iy = rr / ep.dIW, ix = rr % ep.dIW;
                        const int sub = cg / ep.dC, co = cg - sub * ep.dC;
                        const int dy = sub / ep.ds, dx = sub - dy * ep.ds;
                        const size_t opix = ((size_t)b * ep.dIH * ep.ds + (size_t)iy * ep.ds + dy) * (ep.dIW * ep.ds) +
                                            (size_t)ix * ep.ds + dx;
                        o = ep.out + opix * ep.out_ld + co;
                    }
                    if (vec && cg + 3 < p.Cout) {
                        *reinterpret_cast<float4*>(o) = v;
                    } else {
                        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            if (cg + j < p.Cout) o[j] = e[j];
                    }
                }
            }
        } else {
            // NCHW planes and pixel shuffles with a channel count that is not a multiple of 4: one element per
            // thread, consecutive threads on consecutive rows (= consecutive pixels of an NCHW plane)
            for (int idx = tid; idx < GT_ROWS * BN; idx += GT_CONV_THREADS) {
                const int r = idx % GT_ROWS, cl = idx / GT_ROWS, c = col0 + cl;
                const int64_t n = rown[r];
                if (n < 0 || c >= p.Cout) continue;
                float x = stg[r * SLD + cl];
                if (ep.residual) x += ep.residual[(size_t)n * ep.res_ld + c];
                x = apply_act(x, ep.act, ep.slope);
                if (ep.mode == 1) {
                    const int64_t b = n / ep.plane, pix = n % ep.plane;
                    ep.out[((size_t)b * p.Cout + c) * ep.plane + pix] = x;
                } else {
                    const int64_t per = (int64_t)ep.dIH * ep.dIW;
                    const int64_t b = n / per;
                    const int rr = (int)(n % per);
                    const int iy = rr / ep.dIW, ix = rr % ep.dIW;
                    const int sub = c / ep.dC, co = c - sub * ep.dC;
                    const int dy = sub / ep.ds, dx = sub - dy * ep.ds;
                    const size_t opix = ((size_t)b * ep.dIH * ep.ds + (size_t)iy * ep.ds + dy) * (ep.dIW * ep.ds) +
                                        (size_t)ix * ep.ds + dx;
                    ep.out[opix * ep.out_ld + co] = x;
                }
            }
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)ptr;
    }
    return fn;
}

// fp32 tensor map with SWIZZLE_128B (inner box = 32 floats = 128 B), zero OOB fill
static int make_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) O3DML_FAIL(O3DML_ERR_CUDA, "linear_tc: cuTensorMapEncodeTiled is not available from the driver");
    cuuint64_t d[5], s[4];
    cuuint32_t b[5], e[5];
    for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; e[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), d, s, b, e,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) O3DML_FAIL(O3DML_ERR_CUDA, "linear_tc: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return O3DML_OK;
}

template <int BN, bool GATHER, bool LITE = false>
static int gemm_tc_launch_bn(const GemmTcParams& p, unsigned grid_x, cudaStream_t st) {
    using C = GtCfg<BN, LITE>;
    dim3 grid(grid_x, (unsigned)(p.Npad / BN));
    O3DML_CUDA(launch<gemm_tc_kernel<BN, GATHER, LITE>>(grid, gt_threads<GATHER>(), C::SMEM, st, p));
    return O3DML_OK;
}

constexpr int GT_LITE_MAX_SLICES = 16;   // longest product, in 32-channel k-slices, that runs on the LITE kernels

static int gemm_tc_launch(GemmTcParams& p, const void* wimg, int k_pad, int n_pad, cudaStream_t st) {
    p.Kpad = k_pad;
    p.Npad = n_pad;
    O3DML_CHECK(n_pad >= p.Cout, "linear_tc: weight image has fewer rows than out_channels");
    if (p.N <= 0 || p.Cout <= 0) return O3DML_OK;
    O3DML_CHECK(p.Kpad % GT_KS == 0 && p.Kpad >= p.K, "linear_tc: weight image K padding must be a multiple of 32");
    O3DML_CHECK(p.Npad == 32 || p.Npad == 64 || p.Npad % 128 == 0,
                "linear_tc: weight image rows must be padded to 32, 64 or a multiple of 128");
    int bn = p.Npad == 32 ? 32 : (p.Npad == 64 ? 64 : 128);
    bool any_gather = false;
    if (p.mode == 0)
        for (int s = 0; s < p.nsrc; ++s) any_gather = any_gather || p.src[s].index != nullptr;
    const int sms = device_sm_count();
    int64_t row_tiles = ceil_div<int64_t>(p.N, GT_ROWS);
    if (p.mode == 1) {
        int best_tiles = 1 << 30;
        for (int l = 0; l <= 7; ++l) best_tiles = std::min(best_tiles, ceil_div(p.OW, 1 << l) * ceil_div(p.OH, GT_ROWS >> l));
        row_tiles = (p.N / ((int64_t)p.OH * p.OW)) * best_tiles;
    }
    // products of plain row sources, at most 16 k-slices long, that fill the SMs more than once as 64-column tiles run on
    // the LITE kernels, two CTAs per SM (GtCfg); the convolutions (K = 9 C) stay on the one-CTA-per-SM kernels
    const bool lite = p.mode == 0 && !any_gather && p.Kpad / GT_KS <= GT_LITE_MAX_SLICES &&
                      row_tiles * (p.Npad / (bn == 32 ? 32 : 64)) > sms;
    if (lite && bn == 128) bn = 64;
    // a grid that fills less than half of the SMs (PointPillars block 3: 27 x 2 CTAs; one cloud per GPU: 6 - 88)
    // runs as 64-column tiles instead: twice the CTAs, each with half the tensor-core work per slice
    if (bn == 128 && 2 * row_tiles * (p.Npad / 128) <= sms) bn = 64;
    {   // weight image: fp32 [2 * Npad][Kpad] (TF32 hi rows, then lo rows)
        const uint64_t dims[2] = {(uint64_t)p.Kpad, (uint64_t)2 * p.Npad};
        const uint64_t str[1] = {(uint64_t)p.Kpad * 4};
        const uint32_t box[2] = {GT_KS, (uint32_t)bn};
        int rc = make_map(&p.mapB, wimg, 2, dims, str, box);
        if (rc) return rc;
    }
    bool gather = false;
    unsigned grid_x;
    if (p.mode == 0) {
        grid_x = (unsigned)ceil_div<int64_t>(p.N, GT_ROWS);
        for (int s = 0; s < p.nsrc; ++s) {
            if (p.src[s].index) { gather = true; continue; }
            const uint64_t rows = (uint64_t)(p.src[s].rows > 0 ? p.src[s].rows : p.N);
            const uint64_t dims[2] = {(uint64_t)p.src[s].channels, rows};
            const uint64_t str[1] = {(uint64_t)p.src[s].ld * 4};
            const uint32_t box[2] = {GT_KS, GT_ROWS};
            int rc = make_map(&p.mapA[s], p.src[s].data, 2, dims, str, box);
            if (rc) return rc;
        }
    } else {
        // patch of output pixels per CTA: PW x PH = 128, the shape with the fewest tiles
        int best = -1, best_tiles = 0;
        for (int l = 0; l <= 7; ++l) {
            const int pw = 1 << l, ph = GT_ROWS >> l;
            const int tiles = ceil_div(p.OW, pw) * ceil_div(p.OH, ph);
            if (best < 0 || tiles < best_tiles || (tiles == best_tiles && pw >= 8 && (1 << best) < 8)) {
                best = l;
                best_tiles = tiles;
            }
        }
        p.lpw = best;
        p.PH = GT_ROWS >> best;
        p.tiles_x = ceil_div(p.OW, 1 << best);
        p.tiles_y = ceil_div(p.OH, p.PH);
        const int64_t batch = p.N / ((int64_t)p.OH * p.OW);
        grid_x = (unsigned)(batch * p.tiles_x * p.tiles_y);
        const uint32_t box[4] = {GT_KS, (uint32_t)(1 << best), (uint32_t)p.PH, 1};
        const float* in = p.src[0].data;
        if (p.stride == 1) {
            const uint64_t dims[4] = {(uint64_t)p.C, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)batch};
            const uint64_t str[3] = {(uint64_t)p.C * 4, (uint64_t)p.W * p.C * 4, (uint64_t)p.H * p.W * p.C * 4};
            int rc = make_map(&p.mapA[0], in, 4, dims, str, box);
            if (rc) return rc;
        } else {
            for (int py = 0; py < 2; ++py)
                for (int px = 0; px < 2; ++px) {
                    const uint64_t wp = (uint64_t)(p.W - px + 1) / 2, hp = (uint64_t)(p.H - py + 1) / 2;
                    if (wp == 0 || hp == 0) {      // a 1-pixel-wide image has no odd columns: never addressed in range
                        p.mapA[py * 2 + px] = p.mapA[0];
                        continue;
                    }
                    const uint64_t dims[4] = {(uint64_t)p.C, wp, hp, (uint64_t)batch};
                    const uint64_t str[3] = {(uint64_t)2 * p.C * 4, (uint64_t)2 * p.W * p.C * 4,
                                             (uint64_t)p.H * p.W * p.C * 4};
                    int rc = make_map(&p.mapA[py * 2 + px], in + ((size_t)py * p.W + px) * p.C, 4, dims, str, box);
                    if (rc) return rc;
                }
        }
    }
    if (gather) {
        if (bn == 32) return gemm_tc_launch_bn<32, true>(p, grid_x, st);
        if (bn == 64) return gemm_tc_launch_bn<64, true>(p, grid_x, st);
        return gemm_tc_launch_bn<128, true>(p, grid_x, st);
    }
    if (lite) {
        if (bn == 32) return gemm_tc_launch_bn<32, false, true>(p, grid_x, st);
        return gemm_tc_launch_bn<64, false, true>(p, grid_x, st);
    }
    if (bn == 32) return gemm_tc_launch_bn<32, false>(p, grid_x, st);
    if (bn == 64) return gemm_tc_launch_bn<64, false>(p, grid_x, st);
    return gemm_tc_launch_bn<128, false>(p, grid_x, st);
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_linear_tc_supported(const o3dml_src_t* srcs, int num_srcs) {
    if (num_srcs < 1 || num_srcs > GT_MAX_SRC) return 0;
    for (int s = 0; s < num_srcs; ++s) {
        const o3dml_src_t& S = srcs[s];
        if (!S.data || S.channels <= 0 || (S.channels & 3) || (S.ld & 3) || (reinterpret_cast<uintptr_t>(S.data) & 15))
            return 0;
        if (s + 1 < num_srcs && (S.channels % GT_KS) != 0) return 0;   // a k-slice never straddles two sources
    }
    return 1;
}

extern "C" int o3dml_linear_tc(int64_t num_rows, const o3dml_src_t* srcs, int num_srcs,
                               const void* weight_image, int k_pad, int n_pad, const float* scale,
                               const float* shift, const float* residual, int residual_ld, int act,
                               float slope, float* out, int out_ld, int out_channels,
                               int out_nchw_plane, void* stream) {
    GemmTcParams p = {};
    p.N = num_rows;
    p.mode = 0;
    p.nsrc = num_srcs;
    int rc = set_srcs("linear_tc", srcs, num_srcs, p.src, p.koff);
    if (rc) return rc;
    O3DML_CHECK(o3dml_linear_tc_supported(srcs, num_srcs),
                "linear_tc: sources need a multiple of 4 channels (32 for all but the last), 16-byte aligned rows");
    rc = set_epilogue("linear_tc", p, weight_image, scale, shift, residual, residual_ld, act, slope, out, out_ld,
                      out_channels, out_nchw_plane);
    if (rc) return rc;
    p.K = p.koff[GT_MAX_SRC];
    return gemm_tc_launch(p, weight_image, k_pad, n_pad, (cudaStream_t)stream);
}

extern "C" int o3dml_conv3x3_nhwc_tc(const float* in, int batch, int H, int W, int C, int stride,
                                     const void* weight_image, int k_pad, int n_pad, const float* scale,
                                     const float* shift, int act, float slope, float* out,
                                     int out_channels, void* stream) {
    GemmTcParams p = {};
    int rc = set_conv3x3("conv3x3_tc", p, in, batch, H, W, C, stride, GT_KS);
    if (!rc) rc = set_epilogue("conv3x3_tc", p, weight_image, scale, shift, nullptr, 0, act, slope, out, out_channels,
                               out_channels, 0);
    if (rc) return rc;
    return gemm_tc_launch(p, weight_image, k_pad, n_pad, (cudaStream_t)stream);
}

extern "C" int o3dml_deconv_nhwc_tc(const float* in, int batch, int H, int W, int C, int stride,
                                    const void* weight_image, int k_pad, int n_pad, const float* scale,
                                    const float* shift, int act, float slope, float* out, int out_ld,
                                    int out_channels, void* stream) {
    GemmTcParams p = {};
    int rc = set_deconv("deconv_tc", p, weight_image, in, batch, H, W, C, stride, scale, shift, act, slope, out, out_ld,
                        out_channels);
    if (rc) return rc;
    O3DML_CHECK((C % 4) == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0, "deconv_tc: C % 4, aligned input");
    return gemm_tc_launch(p, weight_image, k_pad, n_pad, (cudaStream_t)stream);
}
