// tc.cuh -- hand-written Hopper (sm_90a) tensor-core primitives: wgmma, mbarrier, bulk copies (inline PTX).
//
// Operand conventions used by the tensor-core kernels of this library:
//   * 16-bit operands (fp16), K-major, NO swizzle, "chunk-major" canonical layout
//         element (row r, k)  ->  byte  (k / 8) * (ROWS * 16) + r * 16 + (k % 8) * 2
//     i.e. [K/8][ROWS][8 halves]: a thread that owns 8 consecutive k of one row writes ONE
//     16-byte shared store, consecutive rows are consecutive 16-byte words (conflict-free),
//     and the wgmma descriptor is  LBO = ROWS*16 (next 8-wide k chunk), SBO = 128 (next 8 rows).
//   * fp32 operands (TF32), K-major, SWIZZLE_128B (row r, 16-byte chunk c at r*128 + ((c ^ (r & 7)) << 4)),
//     SBO = 1024 (next 8 rows), K advanced by +32 B per k8 step.
//   * wgmma: one warpgroup computes D[64 x N] (+)= A[64 x K] * B[N x K]^T into registers; warp w of the
//     warpgroup owns rows [16w, 16w+16): d[i] is row 16w + lane/4 + 8*((i/2)%2), column 8*(i/4) + 2*(lane%4) + i%2.
//   * 22-bit "3xFP16" precision: x = h1 + h2 with h1 = fp16(x), h2 = fp16(x - h1);
//     A*B ~= A1*B1 + A1*B2 + A2*B1 (three MMAs into the same accumulator).  Relative error
//     ~2^-21 per product, which keeps the 1e-4 parity bar that plain TF32/BF16 cannot
//     (SURVEY.md section 7).  hi + lo represents x to max(|x| 2^-22, 2^-25): lo falls to fp16 subnormals below
//     2^-14 of |x|.  Without range normalisation (lfa_tc.cu) a tensor of scale s keeps 1e-4 of s for s >= ~2^-11.7;
//     from |x| >= 65520 hi is Inf and, like +-Inf and NaN, the split is non-finite (the conversion does not saturate).
//     Measured through lfa_tc on an H100 (tests/test_gpu_lfa_tc.py): agg stays within 1e-4 of float64 for features of
//     scale 2^-12 .. 2^8 with coordinates within 1e2 of the origin (the reference's crop centres the clouds,
//     ml3d/datasets/utils/transforms.py:123); coordinates near 1e3 cost 1.5e-4 at any feature scale.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace o3dml {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}

// 1-D bulk async copy (TMA engine) global -> shared, completion counted in bytes on the mbarrier
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

// generic-proxy shared-memory writes -> visible to the async proxy (tensor core reads)
__device__ __forceinline__ void fence_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// ---- wgmma ------------------------------------------------------------------------------------
// K-major shared-memory matrix descriptor (sm_90 GmmaDescriptor: start[0,14) lbo[16,30) sbo[32,46)
// layout_type[62,64): 0 = no swizzle, 1 = 128-byte swizzle; addresses and offsets in 16-byte units)
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fffu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32;
    return d;
}
// K-major SWIZZLE_128B: rows of 128 B, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3fffu) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// register writes (A fragments, accumulators) -> visible to the next wgmma of this warpgroup
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// fp32 word of a TF32 operand -> (hi, lo): hi keeps the 10 explicit mantissa bits TF32 uses,
// lo = x - hi is exact in fp32 (the tensor core keeps 11 of its <= 13 bits)
__device__ __forceinline__ void split_tf32(uint32_t x, uint32_t& hi, uint32_t& lo) {
    hi = x & 0xFFFFE000u;
    lo = __float_as_uint(__uint_as_float(x) - __uint_as_float(hi));
}

// wgmma_tf32_rs<N>: D[64 x N] (+)= A (registers: the m16n8k8 TF32 fragment of each warp's 16 rows) * B[smem]^T
// wgmma_f16_ss<N>:  D[64 x N] (+)= A[smem] * B[smem]^T, fp16 operands
// scale_d = 0 overwrites D instead of accumulating.
// ---- generated fixed-arity wrappers (one per accumulator width) ----
template <int N> __device__ void wgmma_tf32_rs(float* d, const uint32_t* a, uint64_t bdesc, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_tf32_rs<32>(float* d, const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<64>(float* d, const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<128>(float* d, const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
}
template <int N> __device__ void wgmma_f16_ss(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_f16_ss<16>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(scale_d)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_f16_ss<32>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(scale_d)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_f16_ss<64>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(scale_d)
        : "memory");
}
// wgmma_f16_ss_set<N>: D[64 x N] = A[smem] * B[smem]^T, fp16 operands; the old values of d are not read, so that they
// need not stay live up to the instruction
template <int N> __device__ void wgmma_f16_ss_set(float* d, uint64_t adesc, uint64_t bdesc);
template <> __device__ __forceinline__ void wgmma_f16_ss_set<64>(float* d, uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(0)
        : "memory");
}
// wait until at most N committed wgmma groups of this warpgroup are pending
template <int N> __device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// pins accumulator registers in place around wgmma issue / wait: the compiler may not move their reads or writes across
__device__ __forceinline__ void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// ---- fp32 -> (h1, h2) split -----------------------------------------------------------------
// 8 consecutive-k floats of one row -> two 16-byte words (hi parts, lo parts)
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
    __half2 t = __halves2half2(a, b);  // a -> low 16 bits (lower k)
    return *reinterpret_cast<uint32_t*>(&t);
}
// packed fp32 pair -> fp16 pair (F2FP.F16.F32.PACK_AB): `lo` lands in the low half (lower k).  Not saturating: +-Inf and
// |x| >= 65520 become +-Inf, so that the split of such a value (hi = Inf, lo = x - hi = -Inf or NaN) is non-finite
// instead of a silently clamped +-65504.
__device__ __forceinline__ uint32_t cvt_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
// 3 instructions per element (F2FP, HADD2.F32, FADD, F2FP over pairs) against ~7 of the scalar convert sequence: the
// split is ~15 % of the SIMT instructions of an LFA tile
__device__ __forceinline__ void split8(const float* x, uint4& hi, uint4& lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        h[i] = cvt_f16x2(x[2 * i], x[2 * i + 1]);
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h[i]));
        l[i] = cvt_f16x2(x[2 * i] - f.x, x[2 * i + 1] - f.y);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// ldmatrix.x4.trans: four 8x8 fp16 matrices, lanes 8j .. 8j + 7 addressing the 16-byte rows of matrix j; r[j] holds
// matrix j transposed in the mma fragment layout: lane (g = lane / 4, t = lane % 4) gets elements (row 2t, column g)
// in the low half and (row 2t + 1, column g) in the high half
__device__ __forceinline__ void ldsm_x4_trans(uint32_t* r, uint32_t saddr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(saddr)
                 : "memory");
}

// byte offset of (row, k-chunk) in the chunk-major canonical layout
__device__ __forceinline__ uint32_t op_off(int rows, int r, int kchunk) {
    return (uint32_t)kchunk * (uint32_t)(rows * 16) + (uint32_t)r * 16u;
}

}  // namespace tc
}  // namespace o3dml
