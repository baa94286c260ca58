// Warpgroup MMA (wgmma) primitives for the Hopper tensor cores of sm_90a (inline PTX; descriptor bit layout as in
// CUTLASS cute/arch/mma_sm90_desc.hpp: GMMA::GmmaDescriptor).
#pragma once
#include "nsb_common.cuh"

namespace nsb {
namespace tc {

// Shared-memory matrix descriptor, K-major, no swizzle ("interleave"): the operand is tiled in 8 x 16-byte core
// matrices (8 rows of 8 halfs, 128 contiguous bytes); LBO = byte distance between the two core matrices of one K = 16
// step, SBO = byte distance between consecutive 8-row groups.  Bits: [0,14) address >> 4, [16,30) LBO >> 4,
// [32,46) SBO >> 4, [49,52) base offset = 0, [62,64) layout type = 0 (INTERLEAVE).
__device__ __forceinline__ uint64_t smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((smem_addr >> 4) & 0x3fffu) | ((uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32);
}

// generic-proxy shared-memory writes -> visible to the async proxy (the tensor core reads operands through it)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// orders this thread's earlier register / shared-memory accesses before the wgmma operations that follow
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 64] (+)= A[64 x 16] . B[64 x 16]^T, both operands K-major in shared memory, fp16 in, fp32 accumulate; issued by
// the whole warpgroup.  D fragment: thread t = 32 w + l holds rows 16 w + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1)
// in d[4 j + 2 * (row half) + (column parity)].
__device__ __forceinline__ void mma_m64n64k16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, bool accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"((uint32_t)accumulate)
        : "memory");
}
// D[64 x 16] (+)= A[64 x 16] . B[16 x 16]^T, same fragment layout (j < 2)
__device__ __forceinline__ void mma_m64n16k16(float (&d)[8], uint64_t a_desc, uint64_t b_desc, bool accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a_desc), "l"(b_desc), "r"((uint32_t)accumulate)
        : "memory");
}

// Register-A forms ("RS": A from registers, B from shared memory).  The fp16 A fragment of one k = 16 step is four
// half2 registers: thread t = 32 w + l holds row 16 w + l / 4 in a[0] (columns 2 (l % 4) + {0, 1}) and a[2] (columns
// 8 + 2 (l % 4) + {0, 1}), and row 16 w + l / 4 + 8 in a[1] / a[3] (same columns).  That is the D fragment above: the
// fp32 d[4 j .. 4 j + 3] of 8-column groups j = 2 s and 2 s + 1, converted pairwise to half2, are exactly
//   a[s] = {h2(d[8 s], d[8 s + 1]), h2(d[8 s + 2], d[8 s + 3]), h2(d[8 s + 4], d[8 s + 5]), h2(d[8 s + 6], d[8 s + 7])},
// so one layer's output feeds the next layer's A operand with no data movement between threads.  The A registers must
// be written before the wg_fence that precedes the MMAs reading them (else ptxas serialises the chain, info C7513).
__device__ __forceinline__ void mma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, bool accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"((uint32_t)accumulate)
        : "memory");
}
__device__ __forceinline__ void mma_m64n16k16_rs(float (&d)[8], const uint32_t (&a)[4], uint64_t b_desc, bool accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"((uint32_t)accumulate)
        : "memory");
}

// exactly one lane of a converged warp (the issuing lane of the bulk copies)
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
// half2(relu(lo), relu(hi)), round-to-nearest: the ReLU rides on the conversion
__device__ __forceinline__ uint32_t cvt_relu_h2(float lo, float hi) {
    uint32_t d;
    asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
// sin(x) for |x| up to a few thousand: two-constant Cody-Waite reduction to [-pi, pi] (k * 2pi_hi is exact inside the
// FMA), then MUFU.SIN (abs error < 4e-7 there).  The result feeds an fp16 MMA operand (spacing 4.9e-4 near 1).
__device__ __forceinline__ float sin_reduced(float x) {
    const float k = rintf(x * 0.15915494309189535f);
    float r = fmaf(-k, 6.2831854820251465f, x);
    r = fmaf(-k, -1.7484555314695172e-07f, r);
    return __sinf(r);
}

}  // namespace tc
}  // namespace nsb
