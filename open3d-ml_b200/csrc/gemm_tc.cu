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
//     which is the convolution padding; stride-2 convolutions use four parity maps; the 3x3x3 convolution is the
//     same with a 5-D {C, Z, Y, X, B} map, the rank limit of the TMA unit, and a PZ x PY x PX box of output voxels),
//   * gathered sources (index / batch-relative index / shadow rows) by 16-byte cp.async into the same
//     128-byte-swizzled layout,
//   * the weight slices (hi and lo image) by two more tensor copies.
// The two consumer warpgroups (64 rows each) read their A fragments straight from the swizzled tile into
// registers, split them there (hi = x & mask, lo = x - hi) and issue register-A wgmma against the W hi / lo
// tiles in shared memory: the split never goes back to shared memory.
// Shared-memory layout: K-major, SWIZZLE_128B (row r, 16-byte chunk c at r*128 + ((c ^ (r & 7)) << 4)),
// descriptors with SBO = 1024, K advanced by +32 B per wgmma (K = 8 TF32).
//
// Table mode (the sparse convolutions): out[m] = sum over the kernel cells c of W_c^T act(x[table[m, c]]), K = cells x
// Cin padded to 32.  The loaders gather each 32-channel slice of a cell from the row the table names (a shadow id
// reads zeros); the (tile, cell) pairs whose 128 rows are all shadow are skipped.  The optional prologue act(x) =
// relu(pre_scale * x + pre_shift) is applied by the consumers in registers before the split, and keeps shadow rows at
// zero: an empty cell contributes nothing, not act(0).  The weighted instances (o3dml_sparse_conv_weighted_tc) also
// scale every entry by a float table parallel to the neighbour table, x' = w[m, c] * act(x), read once per (row, cell)
// where the consumers test the entry for a shadow id; a shadow entry stays zero whatever its weight.
//
// Every GT_FLUSH slices the wgmma accumulator is folded into a second fp32 register set with
// round-to-nearest adds, so that long products do not rely on the tensor core's internal accumulation.
#include "../../include/o3dml_b200.h"
#include "dense.cuh"
#include "tc.cuh"
#include <cuda.h>
#include <type_traits>

namespace o3dml {

constexpr int GT_ROWS = 128;
constexpr int GT_KS = 32;        // fp32 channels per k-slice (= one 128-byte swizzle row)
constexpr int GT_FLUSH = 4;      // k-slices (128 channels = 48 accumulating MMAs) per register accumulation chunk
constexpr int GT_MAX_SRC = 3;
constexpr int GT_TABLE_MAX_CELLS = 512;   // table mode: kernel cells of one contraction (the list fits the rowptr slots)
constexpr int GT_CONV_THREADS = 256;   // warps 0-7: the two consumer warpgroups
constexpr int GT_LOADERS = 128;        // warps 8-11 (GATHER kernels only)
constexpr int GT_A_BYTES = GT_ROWS * 128;

struct alignas(64) GemmTcParams {
    CUtensorMap mapA[4];   // rows mode: one per identity source; conv: stride 1 -> [0], stride 2 -> parity (py*2+px)
    CUtensorMap mapB;      // {Kpad, 2*Npad}: hi rows [0, Npad), lo rows [Npad, 2*Npad)
    int64_t N;
    int K, Kpad, Cout, Npad;
    int mode;  // 0 rows, 1 conv3x3, 2 conv3x3x3, 3 table
    int nsrc;
    o3dml_src_t src[GT_MAX_SRC];
    int koff[GT_MAX_SRC + 1];
    int H, W, OH, OW, stride, C;
    int lpw, PH, tiles_x, tiles_y;   // conv: patch = (1 << lpw) x PH output pixels per CTA
    int X, Y, Z, lpz, lpy, tiles_z;  // conv3x3x3: box = (1 << lpz) x (1 << lpy) x (128 >> (lpz + lpy)) output voxels, z fastest
    DenseEpilogue ep;
    int cells;                              // table mode: src[0] = features + table (index, index_ld), C = Cin padded to 32
    const float* pre_scale;                 // table mode prologue (both or neither)
    const float* pre_shift;
    const float* entry_weight;              // table mode, weighted instances: float [N, weight_ld], parallel to the table
    int weight_ld;
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
__device__ __forceinline__ void tma_load_5d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
        "[%2];" ::"r"(smem_dst),
        "l"(map), "r"(tc::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// table mode: the feature row that row n of the output reads in kernel cell `cell`, nullptr for a shadow id
__device__ __forceinline__ const float* table_row(const GemmTcParams& p, int64_t n, int cell) {
    if (n >= p.N) return nullptr;
    const o3dml_src_t& S = p.src[0];
    const int64_t r = ((const int32_t*)S.index)[n * S.index_ld + cell];
    return (r < 0 || r >= S.rows) ? nullptr : S.data + (size_t)r * S.ld;
}

// table mode: the factor of an entry, its weight in the WEIGHTED instances and a liveness flag in the others
template <bool WEIGHTED>
using TableFactor = typename std::conditional<WEIGHTED, float, bool>::type;

// table mode: the factor of the entry that row n reads in kernel cell `cell`, 0 (false) for a shadow entry or past the
// last row
template <bool WEIGHTED>
__device__ __forceinline__ TableFactor<WEIGHTED> table_entry(const GemmTcParams& p, int64_t n, int cell) {
    if (!table_row(p, n, cell)) return 0;
    if constexpr (WEIGHTED) return __ldg(p.entry_weight + n * p.weight_ld + cell);
    else return true;
}

// table mode: element x of input channel ch as the consumers multiply it, w * relu(pre_scale * x + pre_shift), or w * x
// without a prologue, 0 past Cin.  w is table_entry's factor; outside the WEIGHTED instances it is a liveness flag and
// selects, so that a live entry passes exactly act(x) and a shadow one exactly 0 without reading the prologue.
template <bool WEIGHTED>
__device__ __forceinline__ float table_prologue(const GemmTcParams& p, float x, int ch, TableFactor<WEIGHTED> w) {
    if (ch >= p.src[0].channels || (!WEIGHTED && !w)) return 0.f;
    const float a = p.pre_scale ? fmaxf(fmaf(x, __ldg(p.pre_scale + ch), __ldg(p.pre_shift + ch)), 0.f) : x;
    return WEIGHTED ? w * a : a;
}

// The outputs of one CTA: 128 consecutive rows from row0 (rows and table mode), a (1 << lpw) x PH patch of output pixels
// of image cb from (oy0, ox0) (conv3x3) or a PZ x PY x PX box of output voxels of grid cb from (ox0, oy0, oz0)
// (conv3x3x3); set_tiles chooses the patch and box shapes
struct GtTile {
    int64_t row0;
    int cb, oy0, ox0, oz0;
};

__device__ __forceinline__ GtTile gt_tile(const GemmTcParams& p) {
    GtTile t = {(int64_t)blockIdx.x * GT_ROWS, 0, 0, 0, 0};
    if (p.mode == 1) {
        const int per = p.tiles_x * p.tiles_y;
        t.cb = blockIdx.x / per;
        const int i = blockIdx.x - t.cb * per;
        t.oy0 = (i / p.tiles_x) * p.PH;
        t.ox0 = (i % p.tiles_x) << p.lpw;
    } else if (p.mode == 2) {
        const int per = p.tiles_x * p.tiles_y * p.tiles_z;
        t.cb = blockIdx.x / per;
        const int i = blockIdx.x - t.cb * per, ixy = i / p.tiles_z;
        t.oz0 = (i - ixy * p.tiles_z) << p.lpz;
        t.oy0 = (ixy % p.tiles_y) << p.lpy;
        t.ox0 = (ixy / p.tiles_y) * (GT_ROWS >> (p.lpz + p.lpy));
    }
    return t;
}

// the output row of row m of the tile, -1 past the output
template <bool TABLE>
__device__ __forceinline__ int64_t gt_out_row(const GemmTcParams& p, const GtTile& t, int m) {
    if (TABLE || p.mode == 0) return t.row0 + m < p.N ? t.row0 + m : -1;
    if (p.mode == 1) {
        const int oy = t.oy0 + (m >> p.lpw), ox = t.ox0 + (m & ((1 << p.lpw) - 1));
        return (oy < p.OH && ox < p.OW) ? ((int64_t)t.cb * p.OH + oy) * p.OW + ox : -1;
    }
    const int oz = t.oz0 + (m & ((1 << p.lpz) - 1)), oy = t.oy0 + ((m >> p.lpz) & ((1 << p.lpy) - 1));
    const int ox = t.ox0 + (m >> (p.lpz + p.lpy));
    return (ox < p.X && oy < p.Y && oz < p.Z) ? (((int64_t)t.cb * p.X + ox) * p.Y + oy) * p.Z + oz : -1;
}

// The tensor copy of A slice `sl` into dst: from identity source sidx (rows mode), else from the convolution tap the
// slice belongs to, the tile shifted by the tap (taps in the order of the weight rows)
__device__ __forceinline__ void tma_load_a(const GemmTcParams& p, const GtTile& t, int sl, int sidx, uint32_t dst,
                                           uint64_t* bar) {
    if (p.mode == 0) {
        tma_load_2d(dst, &p.mapA[sidx], sl * GT_KS - p.koff[sidx], (int)t.row0, bar);
        return;
    }
    const int spt = p.C / GT_KS;                      // slices per tap
    const int tap = sl / spt, cc = (sl - tap * spt) * GT_KS;
    if (p.mode == 2) {   // tap (kx * 3 + ky) * 3 + kz
        const int dx = tap / 9, dy = (tap - dx * 9) / 3, dz = tap - dx * 9 - dy * 3;
        tma_load_5d(dst, &p.mapA[0], cc, t.oz0 - 1 + dz, t.oy0 - 1 + dy, t.ox0 - 1 + dx, t.cb, bar);
        return;
    }
    const int dy = tap / 3, dx = tap - dy * 3;
    if (p.stride == 1) {
        tma_load_4d(dst, &p.mapA[0], cc, t.ox0 - 1 + dx, t.oy0 - 1 + dy, t.cb, bar);
    } else {   // input pixel 2*o - 1 + d: odd parity for d = 0 (coordinate o - 1) and d = 2 (o)
        // A 1-pixel-wide (-high) image has no odd columns (rows), and its odd map is the even one (make_a_maps).  Its
        // only output column (row) is 0, and tap d = 2 then reads the padding: coordinate -1, as for d = 0, which the
        // TMA unit fills with zeros.
        const int py = dy != 1, px = dx != 1;
        const int x = t.ox0 - (dx == 0 || (dx == 2 && p.W == 1));
        const int y = t.oy0 - (dy == 0 || (dy == 2 && p.H == 1));
        tma_load_4d(dst, &p.mapA[py * 2 + px], cc, x, y, t.cb, bar);
    }
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

template <int BN, bool GATHER, bool LITE, bool TABLE, bool WEIGHTED>
__global__ void __launch_bounds__(gt_threads<GATHER>(), LITE ? 2 : 1)
gemm_tc_kernel(const __grid_constant__ GemmTcParams p) {
    static_assert(TABLE || !WEIGHTED, "entry weights belong to table mode");
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
    const GtTile tile = gt_tile(p);
    const int64_t row0 = tile.row0;

    // ---- per-row bookkeeping
    for (int m = tid; m < GT_ROWS; m += blockDim.x) rown[m] = gt_out_row<TABLE>(p, tile, m);
    for (int i = tid; i < BN; i += blockDim.x) {      // per-column epilogue constants: read once, not per element
        const int c = col0 + i;
        s_scale[i] = (ep.scale && c < p.Cout) ? ep.scale[c] : 1.f;
        s_shift[i] = (ep.shift && c < p.Cout) ? ep.shift[c] : 0.f;
    }
    // table mode: act[] lists the kernel cells that some row of this tile reads, act[GT_TABLE_MAX_CELLS] counts them
    int* act = reinterpret_cast<int*>(rowptr);
    if (TABLE) {
        for (int c = tid; c < p.cells; c += blockDim.x) act[c] = 0;
        __syncthreads();
        for (int i = tid; i < p.cells * GT_ROWS; i += blockDim.x) {
            const int m = i / p.cells, c = i - m * p.cells;
            if (table_row(p, row0 + m, c)) act[c] = 1;
        }
        __syncthreads();
        if (tid == 0) {
            int k = 0;
            for (int c = 0; c < p.cells; ++c)
                if (act[c]) act[k++] = c;
            act[GT_TABLE_MAX_CELLS] = k;
        }
    } else if (GATHER) {
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

    const int spc = p.C / GT_KS;                      // table mode: slices per kernel cell
    const int nsl = TABLE ? act[GT_TABLE_MAX_CELLS] * spc : p.Kpad / GT_KS;
    const uint32_t stage0 = tc::smem_u32(stages);

    if (warp >= GT_PRODUCER_WARP) {
        // ================================================================= TMA producer (+ gather loaders)
        const int rt = tid - GT_CONV_THREADS;                   // loader index; 0 is also the producer
        if (GATHER || rt == 0) {
            if (rt == 0) tma_prefetch_desc(&p.mapB);
            // loader rt fills 16-byte chunk rt & 7 of rows (rt >> 3) + 16 jj; table mode reads the rows of a cell's
            // table entries at its first slice and keeps them here for the others
            const float* cell_row[(GT_ROWS * 8) / GT_LOADERS] = {};
            int sidx = 0;                                       // the source of the slice (rows mode; table mode: 0)
            for (int sl = 0; sl < nsl; ++sl) {
                const int stage = sl % S, use = sl / S;
                if (use >= 1) tc::mbar_wait(&empty_bar[stage], (use - 1) & 1);
                int k0 = sl * GT_KS, j = 0, cell = 0;          // weight row; table mode: slice j of kernel cell `cell`
                bool a_tma = !TABLE;                            // an identity source or convolution tap
                if (TABLE) {
                    const int ci = sl / spc;
                    j = sl - ci * spc;
                    cell = act[ci];
                    k0 = cell * p.C + j * GT_KS;
                } else if (p.mode == 0) {
                    while (sidx + 1 < p.nsrc && k0 >= p.koff[sidx + 1]) ++sidx;
                    a_tma = p.src[sidx].index == nullptr;
                }
                const uint32_t ah = stage0 + (uint32_t)stage * C::STAGE;
                if (rt == 0) {
                    const uint32_t bh = ah + GT_A_BYTES;
                    mbar_arrive_expect_tx(&full_bar[stage], 2 * C::B_BYTES + (a_tma ? GT_A_BYTES : 0));
                    tma_load_2d(bh, &p.mapB, k0, col0, &full_bar[stage]);
                    tma_load_2d(bh + C::B_BYTES, &p.mapB, k0, p.Npad + col0, &full_bar[stage]);
                    if (a_tma) tma_load_a(p, tile, sl, sidx, ah, &full_bar[stage]);
                }
                if (!GATHER) continue;
                if (a_tma) {
                    mbar_arrive(&full_bar[stage]);
                    continue;
                }
                const int kloc = TABLE ? j * GT_KS : k0 - p.koff[sidx];   // first channel of the slice in its rows
                const int cs = p.src[sidx].channels;
#pragma unroll
                for (int jj = 0; jj < (GT_ROWS * 8) / GT_LOADERS; ++jj) {     // 8 consecutive lanes = one row's 128 B
                    const int item = rt + jj * GT_LOADERS;
                    const int m = item >> 3, c = item & 7;
                    if (TABLE && j == 0) cell_row[jj] = table_row(p, row0 + m, cell);
                    const float* base = TABLE ? cell_row[jj] : rowptr[sidx * GT_ROWS + m];
                    const int kk = kloc + c * 4;
                    // zero past the channels; a gathered source has a multiple of 4 (o3dml_linear_tc_supported)
                    const int bytes = base == nullptr || kk >= cs ? 0 : TABLE ? 4 * min(4, cs - kk) : 16;
                    cp_async16(ah + (uint32_t)m * 128u + (uint32_t)((c ^ (m & 7)) << 4),
                               bytes ? (const void*)(base + kk) : (const void*)p.src[0].data, bytes);
                }
                cp_async_arrive(&full_bar[stage]);
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
        const bool prologue = TABLE && (WEIGHTED || p.pre_scale);
        TableFactor<WEIGHTED> w[2] = {1, 1};   // table prologue: table_entry of rows r0 and r0 + 8 in this cell
        for (int s = 0; s < nsl; ++s) {
            const int stage = s % S, use = s / S;
            int ch0 = 0;                   // table prologue: first input channel of this slice
            if (prologue) {
                const int ci = s / spc, j = s - ci * spc;
                ch0 = j * GT_KS;
                if (j == 0) {
                    w[0] = table_entry<WEIGHTED>(p, row0 + r0, act[ci]);
                    w[1] = table_entry<WEIGHTED>(p, row0 + r0 + 8, act[ci]);
                }
            }
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
                    uint32_t x = *reinterpret_cast<const uint32_t*>(
                        a_tile + r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4);
                    if (prologue) x = __float_as_uint(table_prologue<WEIGHTED>(p, __uint_as_float(x), ch0 + k, w[e & 1]));
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
                    __builtin_assume(ep.mode != 1);
                    float* o = ep.out + out_offset(ep, nr, cg, p.Cout);
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
                __builtin_assume(ep.mode != 0);
                ep.out[out_offset(ep, n, c, p.Cout)] = apply_act(x, ep.act, ep.slope);
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

// The weight image's map: fp32 [2 * Npad][Kpad] (TF32 hi rows, then lo rows), a box of 32 channels x BN columns
static int make_b_map(GemmTcParams& p, const void* wimg, int bn) {
    const uint64_t dims[2] = {(uint64_t)p.Kpad, (uint64_t)2 * p.Npad};
    const uint64_t str[1] = {(uint64_t)p.Kpad * 4};
    const uint32_t box[2] = {GT_KS, (uint32_t)bn};
    return make_map(&p.mapB, wimg, 2, dims, str, box);
}

// The A operand's maps, whose box is one slice of the CTA's tile: rows mode a 2-D {channels, rows} map per identity
// source; conv3x3 a 4-D {C, W, H, B} map (stride 1) or one per (row, column) parity of the input (stride 2); conv3x3x3 a
// 5-D {C, Z, Y, X, B} map.  Gathered sources and table mode have none.
static int make_a_maps(GemmTcParams& p) {
    const float* in = p.src[0].data;
    if (p.mode == 0) {
        for (int s = 0; s < p.nsrc; ++s) {
            if (p.src[s].index) continue;
            const uint64_t rows = (uint64_t)(p.src[s].rows > 0 ? p.src[s].rows : p.N);
            const uint64_t dims[2] = {(uint64_t)p.src[s].channels, rows};
            const uint64_t str[1] = {(uint64_t)p.src[s].ld * 4};
            const uint32_t box[2] = {GT_KS, GT_ROWS};
            int rc = make_map(&p.mapA[s], p.src[s].data, 2, dims, str, box);
            if (rc) return rc;
        }
    } else if (p.mode == 1) {
        const int64_t batch = p.N / ((int64_t)p.OH * p.OW);
        const uint32_t box[4] = {GT_KS, (uint32_t)(1 << p.lpw), (uint32_t)p.PH, 1};
        if (p.stride == 1) {
            const uint64_t dims[4] = {(uint64_t)p.C, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)batch};
            const uint64_t str[3] = {(uint64_t)p.C * 4, (uint64_t)p.W * p.C * 4, (uint64_t)p.H * p.W * p.C * 4};
            return make_map(&p.mapA[0], in, 4, dims, str, box);
        }
        for (int py = 0; py < 2; ++py)
            for (int px = 0; px < 2; ++px) {
                const uint64_t wp = (uint64_t)(p.W - px + 1) / 2, hp = (uint64_t)(p.H - py + 1) / 2;
                if (wp == 0 || hp == 0) {      // no odd columns (rows): the producer reads it at -1 only
                    p.mapA[py * 2 + px] = p.mapA[0];
                    continue;
                }
                const uint64_t dims[4] = {(uint64_t)p.C, wp, hp, (uint64_t)batch};
                const uint64_t str[3] = {(uint64_t)2 * p.C * 4, (uint64_t)2 * p.W * p.C * 4, (uint64_t)p.H * p.W * p.C * 4};
                int rc = make_map(&p.mapA[py * 2 + px], in + ((size_t)py * p.W + px) * p.C, 4, dims, str, box);
                if (rc) return rc;
            }
    } else if (p.mode == 2) {
        const int64_t batch = p.N / ((int64_t)p.X * p.Y * p.Z);
        const uint32_t box[5] = {GT_KS, 1u << p.lpz, 1u << p.lpy, (uint32_t)(GT_ROWS >> (p.lpz + p.lpy)), 1};
        const uint64_t dims[5] = {(uint64_t)p.C, (uint64_t)p.Z, (uint64_t)p.Y, (uint64_t)p.X, (uint64_t)batch};
        const uint64_t str[4] = {(uint64_t)p.C * 4, (uint64_t)p.Z * p.C * 4, (uint64_t)p.Y * p.Z * p.C * 4,
                                 (uint64_t)p.X * p.Y * p.Z * p.C * 4};
        return make_map(&p.mapA[0], in, 5, dims, str, box);
    }
    return O3DML_OK;
}

// Chooses the outputs one CTA owns (GtTile) and returns how many CTAs cover the output, batch x tiles per image or grid
// in the convolutions.  conv3x3: a PW x PH = 128 patch of output pixels, the shape with the fewest patches, on a tie the
// first with PW >= 8.  conv3x3x3: a PZ x PY x PX = 128 box of output voxels with power-of-two sides, the shape with the
// fewest boxes, then the most compact one (its 27 shifted copies overlap most in L2), then the longest run along z.
static int64_t set_tiles(GemmTcParams& p) {
    if (p.mode == 1) {
        int best = -1, best_tiles = 0;
        for (int l = 0; (1 << l) <= GT_ROWS; ++l) {
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
        return p.N / ((int64_t)p.OH * p.OW) * p.tiles_x * p.tiles_y;
    }
    if (p.mode == 2) {
        int64_t best_tiles = -1;
        int best_sum = 0;
        for (int lz = 0; (1 << lz) <= GT_ROWS; ++lz)
            for (int ly = 0; (1 << (lz + ly)) <= GT_ROWS; ++ly) {
                const int pz = 1 << lz, py = 1 << ly, px = GT_ROWS >> (lz + ly);
                const int64_t tiles = (int64_t)ceil_div(p.Z, pz) * ceil_div(p.Y, py) * ceil_div(p.X, px);
                const int sum = pz + py + px;
                if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && sum < best_sum) ||
                    (tiles == best_tiles && sum == best_sum && lz > p.lpz)) {
                    best_tiles = tiles;
                    best_sum = sum;
                    p.lpz = lz;
                    p.lpy = ly;
                }
            }
        p.tiles_z = ceil_div(p.Z, 1 << p.lpz);
        p.tiles_y = ceil_div(p.Y, 1 << p.lpy);
        p.tiles_x = ceil_div(p.X, GT_ROWS >> (p.lpz + p.lpy));
        return p.N / ((int64_t)p.X * p.Y * p.Z) * p.tiles_x * p.tiles_y * p.tiles_z;
    }
    return ceil_div<int64_t>(p.N, GT_ROWS);
}

// An instance of gemm_tc_kernel by its template arguments
struct GtInstance {
    int bn;
    bool gather, lite, table, weighted;
    bool operator==(const GtInstance& o) const {
        return bn == o.bn && gather == o.gather && lite == o.lite && table == o.table && weighted == o.weighted;
    }
};

constexpr int GT_LITE_MAX_SLICES = 16;   // longest product, in 32-channel k-slices, that runs on the LITE kernels

// The instance for `row_tiles` CTAs per column tile on `sms` SMs.  BN is the weight image's padded width up to 64 and
// 128 beyond.  Products of plain row sources, at most 16 k-slices long, that fill the SMs more than once as 64-column
// tiles run on the LITE kernels, two CTAs per SM (GtCfg); the convolutions (K = 9 C, 27 C) stay on the one-CTA-per-SM
// kernels.  A 128-column grid that fills at most half of the SMs (PointPillars block 3: 27 x 2 CTAs; one cloud per GPU:
// 6 - 88) runs as 64-column tiles instead: twice the CTAs, each with half the tensor-core work per slice.
static GtInstance choose_instance(const GemmTcParams& p, int64_t row_tiles, int sms) {
    GtInstance i = {p.Npad == 32 ? 32 : (p.Npad == 64 ? 64 : 128), p.mode == 3, false, p.mode == 3,
                    p.entry_weight != nullptr};
    if (p.mode == 0)
        for (int s = 0; s < p.nsrc; ++s) i.gather = i.gather || p.src[s].index != nullptr;
    i.lite = p.mode == 0 && !i.gather && p.Kpad / GT_KS <= GT_LITE_MAX_SLICES &&
             row_tiles * (p.Npad / (i.bn == 32 ? 32 : 64)) > sms;
    if (i.lite && i.bn == 128) i.bn = 64;
    if (i.bn == 128 && 2 * row_tiles * (p.Npad / 128) <= sms) i.bn = 64;
    return i;
}

template <int BN, bool GATHER, bool LITE, bool TABLE, bool WEIGHTED>
static int gemm_tc_launch_bn(const GemmTcParams& p, unsigned grid_x, cudaStream_t st) {
    using C = GtCfg<BN, LITE>;
    dim3 grid(grid_x, (unsigned)(p.Npad / BN));
    O3DML_CUDA(launch<gemm_tc_kernel<BN, GATHER, LITE, TABLE, WEIGHTED>>(grid, gt_threads<GATHER>(), C::SMEM, st, p));
    return O3DML_OK;
}

struct GtEntry {
    GtInstance inst;
    int (*launch)(const GemmTcParams&, unsigned, cudaStream_t);
};

template <int BN, bool GATHER, bool LITE, bool TABLE, bool WEIGHTED>
constexpr GtEntry gt_entry = {{BN, GATHER, LITE, TABLE, WEIGHTED}, gemm_tc_launch_bn<BN, GATHER, LITE, TABLE, WEIGHTED>};

// Every instance that choose_instance can name (tests/gemm_tc_support.py reads this list)
static const GtEntry GT_INSTANCES[] = {
    gt_entry<128, false, false, false, false>, gt_entry<64, false, false, false, false>,
    gt_entry<32, false, false, false, false>,  gt_entry<64, false, true, false, false>,
    gt_entry<32, false, true, false, false>,   gt_entry<128, true, false, false, false>,
    gt_entry<64, true, false, false, false>,   gt_entry<32, true, false, false, false>,
    gt_entry<128, true, false, true, false>,   gt_entry<64, true, false, true, false>,
    gt_entry<32, true, false, true, false>,    gt_entry<128, true, false, true, true>,
    gt_entry<64, true, false, true, true>,     gt_entry<32, true, false, true, true>,
};

static int gemm_tc_launch(GemmTcParams& p, const void* wimg, int k_pad, int n_pad, cudaStream_t st) {
    p.Kpad = k_pad;
    p.Npad = n_pad;
    O3DML_CHECK(n_pad >= p.Cout, "linear_tc: weight image has fewer rows than out_channels");
    if (p.N <= 0 || p.Cout <= 0) return O3DML_OK;
    O3DML_CHECK(p.Kpad % GT_KS == 0 && p.Kpad >= p.K, "linear_tc: weight image K padding must be a multiple of 32");
    O3DML_CHECK(p.Npad == 32 || p.Npad == 64 || p.Npad % 128 == 0,
                "linear_tc: weight image rows must be padded to 32, 64 or a multiple of 128");
    const int64_t row_tiles = set_tiles(p);
    const GtInstance inst = choose_instance(p, row_tiles, device_sm_count());
    int rc = make_b_map(p, wimg, inst.bn);
    if (!rc) rc = make_a_maps(p);
    if (rc) return rc;
    for (const GtEntry& e : GT_INSTANCES)
        if (e.inst == inst) return e.launch(p, (unsigned)row_tiles, st);
    O3DML_FAIL(O3DML_ERR_UNSUPPORTED, "linear_tc: no gemm_tc_kernel instance <%d, %d, %d, %d, %d>", inst.bn,
               (int)inst.gather, (int)inst.lite, (int)inst.table, (int)inst.weighted);
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

extern "C" int o3dml_conv3x3x3_ndhwc_tc(const float* in, int batch, int X, int Y, int Z, int C, const void* weight_image,
                                        int k_pad, int n_pad, const float* scale, const float* shift, int act,
                                        float slope, float* out, int out_channels, void* stream) {
    GemmTcParams p = {};
    int rc = set_conv3x3x3("conv3x3x3_tc", p, in, batch, X, Y, Z, C, GT_KS);
    if (!rc) rc = set_epilogue("conv3x3x3_tc", p, weight_image, scale, shift, nullptr, 0, act, slope, out, out_channels,
                               out_channels, 0);
    if (rc) return rc;
    return gemm_tc_launch(p, weight_image, k_pad, n_pad, (cudaStream_t)stream);
}

// The argument checks and table-mode parameters of both sparse-convolution entries.  Returns O3DML_OK with p.N == 0
// when there is nothing to launch.
static int set_sparse_table(const char* op, GemmTcParams& p, int64_t num_out, const float* features, int64_t num_in,
                            int channels, int features_ld, const int32_t* table, int cells, int table_ld,
                            const float* pre_scale, const float* pre_shift, const void* weight_image, int k_pad,
                            const float* scale, const float* shift, const float* residual, int residual_ld, int act,
                            float slope, float* out, int out_ld, int out_channels) {
    O3DML_CHECK(num_out >= 0 && num_in >= 0 && num_in < ((int64_t)1 << 31), "%s: bad sizes", op);
    O3DML_CHECK(cells >= 1 && cells <= GT_TABLE_MAX_CELLS, "%s: 1..%d kernel cells", op, GT_TABLE_MAX_CELLS);
    if (num_out == 0) return O3DML_OK;
    O3DML_CHECK(features && table && table_ld >= cells, "%s: null features / table or table_ld < cells", op);
    O3DML_CHECK(channels > 0 && features_ld >= channels && (features_ld & 3) == 0 &&
                    (reinterpret_cast<uintptr_t>(features) & 15) == 0,
                "%s: feature rows need a stride that is a multiple of 4 floats and 16-byte alignment", op);
    O3DML_CHECK((pre_scale == nullptr) == (pre_shift == nullptr), "%s: pre_scale and pre_shift go together", op);
    p.mode = 3;
    p.N = num_out;
    p.nsrc = 1;
    p.cells = cells;
    p.C = (channels + GT_KS - 1) / GT_KS * GT_KS;
    p.K = cells * p.C;
    O3DML_CHECK(k_pad == p.K, "%s: the weight image must have cells * pad32(channels) = %d rows", op, p.K);
    p.src[0].data = features;
    p.src[0].index = table;
    p.src[0].rows = num_in;
    p.src[0].channels = channels;
    p.src[0].ld = features_ld;
    p.src[0].index_ld = table_ld;
    p.pre_scale = pre_scale;
    p.pre_shift = pre_shift;
    return set_epilogue(op, p, weight_image, scale, shift, residual, residual_ld, act, slope, out, out_ld, out_channels,
                        0);
}

extern "C" int o3dml_sparse_conv_tc(int64_t num_out, const float* features, int64_t num_in, int channels,
                                    int features_ld, const int32_t* table, int cells, int table_ld,
                                    const float* pre_scale, const float* pre_shift, const void* weight_image,
                                    int k_pad, int n_pad, const float* scale, const float* shift,
                                    const float* residual, int residual_ld, int act, float slope, float* out,
                                    int out_ld, int out_channels, void* stream) {
    GemmTcParams p = {};
    const int rc = set_sparse_table("sparse_conv_tc", p, num_out, features, num_in, channels, features_ld, table, cells,
                                    table_ld, pre_scale, pre_shift, weight_image, k_pad, scale, shift, residual,
                                    residual_ld, act, slope, out, out_ld, out_channels);
    if (rc || p.N == 0) return rc;
    return gemm_tc_launch(p, weight_image, k_pad, n_pad, (cudaStream_t)stream);
}

extern "C" int o3dml_sparse_conv_weighted_tc(int64_t num_out, const float* features, int64_t num_in, int channels,
                                             int features_ld, const int32_t* table, int cells, int table_ld,
                                             const float* pre_scale, const float* pre_shift, const void* weight_image,
                                             int k_pad, int n_pad, const float* scale, const float* shift,
                                             const float* residual, int residual_ld, int act, float slope, float* out,
                                             int out_ld, int out_channels, const float* entry_weight, int weight_ld,
                                             void* stream) {
    GemmTcParams p = {};
    const int rc = set_sparse_table("sparse_conv_weighted_tc", p, num_out, features, num_in, channels, features_ld,
                                    table, cells, table_ld, pre_scale, pre_shift, weight_image, k_pad, scale, shift,
                                    residual, residual_ld, act, slope, out, out_ld, out_channels);
    if (rc || p.N == 0) return rc;
    O3DML_CHECK(entry_weight && weight_ld >= cells, "sparse_conv_weighted_tc: null entry_weight or weight_ld < cells");
    p.entry_weight = entry_weight;
    p.weight_ld = weight_ld;
    return gemm_tc_launch(p, weight_image, k_pad, n_pad, (cudaStream_t)stream);
}
