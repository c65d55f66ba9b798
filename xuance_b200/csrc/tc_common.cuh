// wgmma building blocks shared by the tensor-core kernels (K9-TC qmix_tc.cu, K12 conv_tc.cu), sm_90a: the K-major
// no-swizzle canonical shared-memory layout, the shared-memory matrix descriptor (LBO = 128 B between K-adjacent core
// matrices, SBO between 8-row groups, layout type in bits 62-63), bf16 x bf16 -> fp32 warpgroup MMAs with the accumulator
// in registers, issued by all 128 threads of a warpgroup.
//
// Accumulator fragment of one m64nNk16 wgmma (PTX ISA, "wgmma .m64nNk16 register fragment D"): thread t of the warpgroup
// (warp w = t / 32, lane l) holds the rows 16 w + l / 4 and 16 w + l / 4 + 8; register 4 i + 2 h + e is row (h = 0 | 1),
// column 8 i + 2 (l % 4) + e.  An n64 fragment is two n32 fragments back to back (columns 0-31, 32-63), so the kernels keep
// accumulators as arrays of 32-column blocks of 16 registers.
#pragma once
#include "xb_common.cuh"

namespace xbtc {

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16 &hi, __nv_bfloat16 &lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// byte offset of element (r, k) of a [rows x KP] bf16 operand in the K-major no-swizzle canonical layout:
// core matrix = 8 rows x 8 elements (16 B per row, 128 B per core), K-adjacent cores contiguous (LBO = 128 B),
// 8-row groups SBO = KP/8 * 128 B apart.
__device__ __forceinline__ uint32_t canon_off(int r, int k, int KP) {
    return (uint32_t)((r >> 3) * (KP >> 3) * 128 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
}

// no-swizzle descriptor (layout type 0) of the canonical layout above
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, int KP) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);               // start address
    d |= (uint64_t)((128 >> 4) & 0x3fff) << 16;               // LBO: next core matrix along K
    d |= (uint64_t)((((KP >> 3) * 128) >> 4) & 0x3fff) << 32; // SBO: next 8-row group
    return d;                                                 // layout type 0 (no swizzle), base offset 0
}

// 128-byte-swizzle descriptor (layout type 1, the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x 16] (+)= A . B^T; TA / TB = 1: that operand is MN-major in shared memory
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}

// D[64 x 64]: columns 0-31 in d0, 32-63 in d1
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d0)[16], float (&d1)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d0[0]), "+f"(d0[1]), "+f"(d0[2]), "+f"(d0[3]), "+f"(d0[4]), "+f"(d0[5]), "+f"(d0[6]), "+f"(d0[7]),
          "+f"(d0[8]), "+f"(d0[9]), "+f"(d0[10]), "+f"(d0[11]), "+f"(d0[12]), "+f"(d0[13]), "+f"(d0[14]), "+f"(d0[15]),
          "+f"(d1[0]), "+f"(d1[1]), "+f"(d1[2]), "+f"(d1[3]), "+f"(d1[4]), "+f"(d1[5]), "+f"(d1[6]), "+f"(d1[7]),
          "+f"(d1[8]), "+f"(d1[9]), "+f"(d1[10]), "+f"(d1[11]), "+f"(d1[12]), "+f"(d1[13]), "+f"(d1[14]), "+f"(d1[15])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}

__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 a, __nv_bfloat16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
// split 8 consecutive-k floats of one row and store them as ONE 16-byte core-matrix row each (hi, lo)
__device__ __forceinline__ void store_unit(const float (&x)[8], int r, int k0, int KP, uint8_t *hi, uint8_t *lo) {
    __nv_bfloat16 h[8], l[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) split_bf16(x[i], h[i], l[i]);
    const uint32_t off = canon_off(r, k0, KP);
    *reinterpret_cast<uint4 *>(hi + off) = make_uint4(pack2(h[0], h[1]), pack2(h[2], h[3]), pack2(h[4], h[5]), pack2(h[6], h[7]));
    *reinterpret_cast<uint4 *>(lo + off) = make_uint4(pack2(l[0], l[1]), pack2(l[2], l[3]), pack2(l[4], l[5]), pack2(l[6], l[7]));
}
// the same for two consecutive-k floats (k0 even): one 4-byte store per plane
__device__ __forceinline__ void store_pair(float x0, float x1, int r, int k0, int KP, uint8_t *hi, uint8_t *lo) {
    __nv_bfloat16 h0, l0, h1, l1;
    split_bf16(x0, h0, l0);
    split_bf16(x1, h1, l1);
    const uint32_t off = canon_off(r, k0, KP);
    *reinterpret_cast<uint32_t *>(hi + off) = pack2(h0, h1);
    *reinterpret_cast<uint32_t *>(lo + off) = pack2(l0, l1);
}

}  // namespace xbtc
