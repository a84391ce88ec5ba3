// prims.cu -- device-wide primitives written for this library:
//   * exclusive scan of uint32 arrays (single-block fast path, single-pass decoupled look-back above one tile)
//   * stable LSD radix sort of (uint64 key, uint32 value) pairs, 8 bits per pass
// Both are small-N, latency-bound steps of the voxel / hash-grid builders
// (N = 2e4 .. 3e5 points per call), so they favour few, simple launches over
// peak sort throughput.  All temporary storage comes from the caller.
#include "prims.cuh"

namespace o3dml {

// ------------------------------------------------------------------ scan ----
constexpr int SCAN_THREADS = 1024;
constexpr int SCAN_ITEMS = 4;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// block-wide exclusive scan of one value per thread (1024 threads)
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total,
                                                    uint32_t* warp_sums /*[32]*/) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = warp_sums[lane];
        uint32_t winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += t;
        }
        warp_sums[lane] = winc - w;  // exclusive
        if (lane == 31) *total = winc;
    }
    __syncthreads();
    uint32_t r = warp_sums[warp] + inc - v;
    __syncthreads();
    return r;
}

// One block scans the whole array tile by tile (n <= a few 100k, or the tile sums).
__global__ void __launch_bounds__(SCAN_THREADS)
scan_single_block(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int64_t n,
                  uint32_t* __restrict__ total_out) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t tile_total;
    uint32_t carry = 0;
    for (int64_t base = 0; base < n; base += SCAN_TILE) {
        uint32_t v[SCAN_ITEMS];
        uint32_t s = 0;
        int64_t i0 = base + (int64_t)threadIdx.x * SCAN_ITEMS;
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
            v[j] = (i0 + j < n) ? in[i0 + j] : 0u;
            s += v[j];
        }
        uint32_t ex = block_excl_scan(s, &tile_total, warp_sums) + carry;
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
            if (i0 + j < n) out[i0 + j] = ex;
            ex += v[j];
        }
        carry += tile_total;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total_out) *total_out = carry;
}

// Single-pass scan with decoupled look-back (one launch for any n > one tile): every block takes a tile ticket
// (atomic counter: a block only ever waits for blocks that already hold a lower ticket, i.e. are resident or done),
// publishes its tile aggregate, then walks back over its predecessors' 64-bit status words
// (flag << 32 | value; flag 1 = aggregate, 2 = inclusive prefix) until it meets an inclusive prefix.
// Replaces the single-block multi-tile loop (12 us at 40 k elements: 5 of them per voxelize call) and the
// 3-launch path above 64 k elements.  status[0] is the ticket counter, status[1 + tile] the tile states; the caller's
// temp buffer is zeroed by a memset node in front of the launch.
__global__ void __launch_bounds__(SCAN_THREADS)
scan_lookback(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int64_t n,
              unsigned long long* __restrict__ status, uint32_t* __restrict__ total_out) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t tile_total;
    __shared__ uint32_t s_tile, s_prefix;
    if (threadIdx.x == 0) s_tile = (uint32_t)atomicAdd(&status[0], 1ull);
    __syncthreads();
    const uint32_t tile = s_tile;
    const int64_t i0 = (int64_t)tile * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint32_t s = 0;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        v[j] = (i0 + j < n) ? in[i0 + j] : 0u;
        s += v[j];
    }
    uint32_t ex = block_excl_scan(s, &tile_total, warp_sums);
    if (threadIdx.x == 0) {
        volatile unsigned long long* st = status + 1;
        const uint32_t total = tile_total;
        uint32_t prefix = 0;
        if (tile == 0) {
            st[0] = (2ull << 32) | total;
        } else {
            st[tile] = (1ull << 32) | total;
            __threadfence();
            for (int64_t j = (int64_t)tile - 1; j >= 0; --j) {
                unsigned long long w;
                do { w = st[j]; } while ((w >> 32) == 0ull);
                prefix += (uint32_t)w;
                if ((w >> 32) == 2ull) break;
            }
            st[tile] = (2ull << 32) | (uint32_t)(prefix + total);
        }
        __threadfence();
        s_prefix = prefix;
        if (total_out && (int64_t)(tile + 1) * SCAN_TILE >= n) *total_out = prefix + total;
    }
    __syncthreads();
    ex += s_prefix;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        if (i0 + j < n) out[i0 + j] = ex;
        ex += v[j];
    }
}

void* scan_carve(Workspace& ws, int64_t n) {
    return ws.take<unsigned long long>((size_t)ceil_div<int64_t>(n, SCAN_TILE) + 2);
}

// out may alias in.  total_out (device, optional) receives the grand total.
cudaError_t exclusive_scan_u32(const uint32_t* in, uint32_t* out, int64_t n, uint32_t* total_out,
                               void* temp, cudaStream_t st) {
    if (n <= 0) {
        if (total_out) return cudaMemsetAsync(total_out, 0, sizeof(uint32_t), st);
        return cudaSuccess;
    }
    if (n <= SCAN_TILE) return launch<scan_single_block>(1, SCAN_THREADS, 0, st, in, out, n, total_out);
    const int64_t tiles = ceil_div<int64_t>(n, SCAN_TILE);
    cudaError_t e = cudaMemsetAsync(temp, 0, (size_t)(tiles + 1) * sizeof(unsigned long long), st);
    if (e != cudaSuccess) return e;
    return launch<scan_lookback>((unsigned)tiles, SCAN_THREADS, 0, st, in, out, n, (unsigned long long*)temp, total_out);
}

// ------------------------------------------------------------ radix sort ----
constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_ITERS = 8;                          // keys per thread
constexpr int RS_TILE = RS_THREADS * RS_ITERS;       // 2048 keys per block
constexpr int RS_BINS = 256;

__device__ __forceinline__ uint32_t rs_digit(uint64_t key, int shift) {
    return (uint32_t)(key >> shift) & (RS_BINS - 1);
}

// per-block digit histogram, written digit-major: hist[d * nblk + blk]
__global__ void __launch_bounds__(RS_THREADS)
rs_histogram(const uint64_t* __restrict__ keys, int64_t n, int shift,
             uint32_t* __restrict__ hist, int nblk) {
    __shared__ uint32_t h[RS_BINS];
    h[threadIdx.x] = 0;
    __syncthreads();
    int64_t base = (int64_t)blockIdx.x * RS_TILE;
#pragma unroll
    for (int it = 0; it < RS_ITERS; ++it) {
        int64_t i = base + it * RS_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&h[rs_digit(keys[i], shift)], 1u);
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

// Stable scatter.  Warp w of the block owns the contiguous key range
// [base + w*256, base + (w+1)*256) and walks it 32 keys at a time, so that
// (block, warp, iteration, lane) order equals input order.
__global__ void __launch_bounds__(RS_THREADS)
rs_scatter(const uint64_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
           uint64_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, int64_t n, int shift,
           const uint32_t* __restrict__ hist_scanned, int nblk) {
    __shared__ uint32_t whist[RS_WARPS][RS_BINS];
    __shared__ uint32_t gbase[RS_BINS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < RS_WARPS * RS_BINS; i += RS_THREADS) (&whist[0][0])[i] = 0;
    gbase[threadIdx.x] = hist_scanned[(size_t)threadIdx.x * nblk + blockIdx.x];
    __syncthreads();

    const int64_t wbase = (int64_t)blockIdx.x * RS_TILE + (int64_t)warp * (32 * RS_ITERS);
    uint64_t key[RS_ITERS];
    uint32_t val[RS_ITERS], rank[RS_ITERS], dig[RS_ITERS];
    const uint32_t lt_mask = (1u << lane) - 1u;
#pragma unroll
    for (int it = 0; it < RS_ITERS; ++it) {
        int64_t i = wbase + it * 32 + lane;
        bool valid = i < n;
        key[it] = valid ? keys_in[i] : 0ull;
        val[it] = valid ? (vals_in ? vals_in[i] : (uint32_t)i) : 0u;
        uint32_t d = valid ? rs_digit(key[it], shift) : (uint32_t)(RS_BINS + lane);
        dig[it] = d;
        uint32_t peers = __match_any_sync(0xffffffffu, d);
        int leader = __ffs(peers) - 1;
        uint32_t old = 0;
        if (valid && lane == leader) {
            old = whist[warp][d];
            whist[warp][d] = old + __popc(peers);
        }
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[it] = old + __popc(peers & lt_mask);
        __syncwarp();
    }
    __syncthreads();
    {   // exclusive prefix over the warps, per digit
        uint32_t run = 0;
        const int d = threadIdx.x;
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) {
            uint32_t c = whist[w][d];
            whist[w][d] = run;
            run += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < RS_ITERS; ++it) {
        int64_t i = wbase + it * 32 + lane;
        if (i < n) {
            uint32_t d = dig[it];
            uint32_t dst = gbase[d] + whist[warp][d] + rank[it];
            keys_out[dst] = key[it];
            vals_out[dst] = val[it];
        }
    }
}

RadixSortBufs radix_sort_carve(Workspace& ws, int64_t n) {
    const int64_t bins = (int64_t)RS_BINS * ceil_div<int64_t>(n > 0 ? n : 1, RS_TILE);
    RadixSortBufs b;
    b.keys_a = ws.take<uint64_t>(n);
    b.keys_b = ws.take<uint64_t>(n);
    b.vals_a = ws.take<uint32_t>(n);
    b.vals_b = ws.take<uint32_t>(n);
    b.hist = ws.take<uint32_t>(bins);
    b.scan_tmp = scan_carve(ws, bins);
    return b;
}

// Stable sort of bits [0, num_bits) of the n pairs in (keys_a, vals_a), n <= the n that `b` was carved for.
// vals_are_iota: ignore vals_a on input and use 0..n-1.  Each pass scatters from the (a) buffers into the (b) buffers
// and then swaps the two in `b`, so that the sorted pairs end in (keys_a, vals_a).
cudaError_t radix_sort_pairs(RadixSortBufs& b, bool vals_are_iota, int64_t n, int num_bits, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    int nblk = (int)ceil_div<int64_t>(n, RS_TILE);
    int passes = (num_bits + 7) / 8;
    if (passes < 1) passes = 1;
    for (int p = 0; p < passes; ++p) {
        int shift = 8 * p;
        cudaError_t e = launch<rs_histogram>(nblk, RS_THREADS, 0, st, b.keys_a, n, shift, b.hist, nblk);
        if (e == cudaSuccess) e = exclusive_scan_u32(b.hist, b.hist, (int64_t)RS_BINS * nblk, nullptr, b.scan_tmp, st);
        if (e == cudaSuccess)
            e = launch<rs_scatter>(nblk, RS_THREADS, 0, st, b.keys_a, (p == 0 && vals_are_iota) ? nullptr : b.vals_a,
                                   b.keys_b, b.vals_b, n, shift, b.hist, nblk);
        if (e != cudaSuccess) return e;
        std::swap(b.keys_a, b.keys_b);
        std::swap(b.vals_a, b.vals_b);
    }
    return cudaSuccess;
}

}  // namespace o3dml
