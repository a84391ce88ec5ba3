// common.cuh -- shared helpers for the sm_90a kernels of libo3dml_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <utility>

#define O3DML_OK 0
#define O3DML_ERR_INVALID 1
#define O3DML_ERR_WORKSPACE 2
#define O3DML_ERR_CUDA 3
#define O3DML_ERR_UNSUPPORTED 4

extern "C" void o3dml_set_error(const char* fmt, ...);

#define O3DML_FAIL(code, ...)      \
    do {                           \
        o3dml_set_error(__VA_ARGS__); \
        return (code);             \
    } while (0)

#define O3DML_CHECK(cond, ...)                               \
    do {                                                     \
        if (!(cond)) O3DML_FAIL(O3DML_ERR_INVALID, __VA_ARGS__); \
    } while (0)

#define O3DML_CHECK_WORKSPACE(ws, entry)                                                                    \
    do {                                                                                                    \
        if (!(ws).ok) O3DML_FAIL(O3DML_ERR_WORKSPACE, entry ": workspace too small (%zu needed)", (ws).off); \
    } while (0)

// variadic so that the commas of a template argument list, launch<k<A, B>>(...), need no extra parentheses
#define O3DML_CUDA(...)                                                               \
    do {                                                                              \
        cudaError_t e__ = (__VA_ARGS__);                                              \
        if (e__ != cudaSuccess)                                                       \
            O3DML_FAIL(O3DML_ERR_CUDA, "%s failed: %s (%s:%d)", #__VA_ARGS__,         \
                       cudaGetErrorString(e__), __FILE__, __LINE__);                  \
    } while (0)

namespace o3dml {

constexpr int kNumSMs = 132;  // H100 SXM (fallback when the attribute query fails)

void count_launch();  // adds one to o3dml_launch_count()

// Opts Kernel into `smem` bytes of dynamic shared memory when that is more than the 48 KB default.  The limit is a
// per-device function attribute, so it is set once per device ordinal (a process may drive several GPUs).
// Precondition: every launch of one Kernel asks for the same `smem`.
template <auto Kernel>
cudaError_t opt_in_smem(size_t smem) {
    if (smem <= 48 * 1024) return cudaSuccess;
    static std::atomic<unsigned long long> done{0};  // one bit per device ordinal
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess || dev >= 64) dev = -1;
    if (dev >= 0 && ((done.load(std::memory_order_relaxed) >> dev) & 1ull)) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess && dev >= 0) done.fetch_or(1ull << dev, std::memory_order_relaxed);
    return e;
}

// Every kernel of the library is enqueued here, so that o3dml_launch_count() counts exactly the kernels that were
// enqueued (memsets and copies are not counted).  Returns the launch error; call sites wrap it in O3DML_CUDA so the
// message names the failing launch.  A failed launch is also cleared from cudaGetLastError(), so that a later,
// unrelated check does not report it again.
template <auto Kernel, class... Args>
cudaError_t launch(dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaError_t e = opt_in_smem<Kernel>(smem);
    if (e == cudaSuccess) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = grid;
        cfg.blockDim = block;
        cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        e = cudaLaunchKernelEx(&cfg, Kernel, std::forward<Args>(args)...);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        return e;
    }
    count_launch();
    return cudaSuccess;
}

inline int device_sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess &&
        n > 0)
        return n;
    return kNumSMs;
}

template <typename T>
__host__ __device__ inline T ceil_div(T a, T b) {
    return (a + b - 1) / b;
}

// Bump allocator over a caller-provided workspace, in 256-byte aligned pieces.  Each entry point lays its workspace
// out in one carve function, carve(Workspace&, sizes...): the entry carves the caller's buffer and checks it with
// O3DML_CHECK_WORKSPACE before it enqueues anything, and its *_workspace_bytes returns measure(carve, sizes...).
// `off` adds up every take, whether it fitted or not, so it is both the exact size and what a failed carve needed.
struct Workspace {
    char* base;
    size_t size, off = 0;
    bool ok = true;  // every take so far fitted; a take that does not returns nullptr, as do all that follow it
    Workspace(void* p, size_t n) : base((char*)p), size(n) {}
    template <class Carve, class... Args>
    static size_t measure(Carve carve, Args... args) {  // the bytes carve(ws, args...) takes; hands out no memory
        Workspace ws(nullptr, 0);
        carve(ws, args...);
        return ws.off;
    }
    template <typename T>
    T* take(size_t count) {
        const size_t at = off;
        off += (count * sizeof(T) + 255) / 256 * 256;
        ok = ok && base && off <= size;
        return ok ? (T*)(base + at) : nullptr;
    }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// float32 squared distance with the operation order of the op contract
// (oracle/ops_ref.c sqdist3): ((dx*dx + dy*dy) + dz*dz), no FMA contraction.
__device__ __forceinline__ float sqdist3(float qx, float qy, float qz, float px, float py,
                                         float pz) {
    float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ int64_t load_index(const void* p, int64_t i, int is64) {
    return is64 ? ((const int64_t*)p)[i] : (int64_t)((const int32_t*)p)[i];
}

// The same load with the result left untouched in two 32-bit words: a software-pipelined gather loads the index of a
// later tile and must not compute anything from it before that tile comes up (the sign extension / select of
// load_index is scheduled right behind the load and waits for it).  index_value() resolves it at the point of use.
struct RawIndex {
    int lo, hi;
};
__device__ __forceinline__ void load_index_raw(const void* p, int64_t i, int is64, RawIndex& r) {
    if (is64) {
        const int2 v = ((const int2*)p)[i];
        r.lo = v.x;
        r.hi = v.y;
    } else {
        r.lo = ((const int32_t*)p)[i];
    }
}
__device__ __forceinline__ int64_t index_value(const RawIndex& r, int is64) {
    return is64 ? (int64_t)(((uint64_t)(uint32_t)r.hi << 32) | (uint64_t)(uint32_t)r.lo) : (int64_t)r.lo;
}

// (d0, d1) += a * (b0, b1): two independent IEEE fp32 FMAs (sm_90 has no packed fp32 FMA).
__device__ __forceinline__ void ffma2(float& d0, float& d1, float a, float b0, float b1) {
    d0 = fmaf(a, b0, d0);
    d1 = fmaf(a, b1, d1);
}

// 2^x as ONE MUFU (ex2.approx.ftz, relative error 2^-22).  Softmax weights are taken as
// exp(s - m) = 2^(s * log2e - m * log2e): an FFMA and a MUFU per weight (expf: ~8 instructions, __expf: 5).
constexpr float kLog2e = 1.4426950408889634f;
__device__ __forceinline__ float ex2_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// activation codes shared with the C ABI
enum { ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY = 2 };
__device__ __forceinline__ float apply_act(float v, int act, float slope) {
    if (act == ACT_RELU) return fmaxf(v, 0.f);
    if (act == ACT_LEAKY) return v >= 0.f ? v : v * slope;
    return v;
}

}  // namespace o3dml
