// Hopper warpgroup MMA (wgmma.mma_async, sm_90a): bf16 inputs, fp32 accumulators in registers.
// Accumulator fragment of m64nNk16 for thread t of the warpgroup (w = t / 32, l = t % 32):
//   d[4i + 0..1] -> row 16w + l/4,     columns 8i + 2(l%4) + {0, 1}
//   d[4i + 2..3] -> row 16w + l/4 + 8, same columns
// The A fragment of the register form (k16 slice) uses the same row/column map for columns 0..15, so the accumulator of one
// product converts to the A operand of the next without shared memory (a[0..3] = pairs (d0,d1), (d2,d3), (d4,d5), (d6,d7)).
#pragma once
#include <stdint.h>

namespace br {

// Shared-memory matrix descriptor, 128-byte swizzle (layout type 1 in bits [62,64)).
// K-major: rows of 64 bf16 (128 B), 8-row groups 1024 B apart; advance 16 elements along K with +2 (32 B >> 4).
__device__ __forceinline__ uint64_t wg_desc_k(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// MN-major: rows of 64 MN-contiguous bf16 (one row per K index), 8-row groups `sbo` bytes apart, 64-wide MN blocks `lbo` bytes apart.
__device__ __forceinline__ uint64_t wg_desc_mn(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32) |
           ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across an in-flight wgmma
template <int N>
__device__ __forceinline__ void wg_fence_operand(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// accumulator operand lists: 8 registers at a time
#define BR_WG_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define BR_WG_F16(i) BR_WG_F8(i), BR_WG_F8(i + 8)
#define BR_WG_F32(i) BR_WG_F16(i), BR_WG_F16(i + 16)
#define BR_WG_F64(i) BR_WG_F32(i), BR_WG_F32(i + 32)
#define BR_WG_F128(i) BR_WG_F64(i), BR_WG_F64(i + 64)

template <int N, int TA, int TB> struct WgSS;
template <int N, int TB> struct WgRS;

template <int TA, int TB> struct WgSS<16, TA, TB> {      // D[64 x 16] (+)= A[64 x 16] . B[16 x 16]; TA / TB = 1: MN-major operand
    static __device__ __forceinline__ void run(float (&d)[8], uint64_t a, uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
                     : BR_WG_F8(0) : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgSS<32, TA, TB> {      // D[64 x 32] (+)= A[64 x 16] . B[16 x 32]; TA / TB = 1: MN-major operand
    static __device__ __forceinline__ void run(float (&d)[16], uint64_t a, uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
                     : BR_WG_F16(0) : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgSS<64, TA, TB> {      // D[64 x 64] (+)= A[64 x 16] . B[16 x 64]; TA / TB = 1: MN-major operand
    static __device__ __forceinline__ void run(float (&d)[32], uint64_t a, uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
                     : BR_WG_F32(0) : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgSS<128, TA, TB> {      // D[64 x 128] (+)= A[64 x 16] . B[16 x 128]; TA / TB = 1: MN-major operand
    static __device__ __forceinline__ void run(float (&d)[64], uint64_t a, uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
                     : BR_WG_F64(0) : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgSS<256, TA, TB> {      // D[64 x 256] (+)= A[64 x 16] . B[16 x 256]; TA / TB = 1: MN-major operand
    static __device__ __forceinline__ void run(float (&d)[128], uint64_t a, uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n}\n"
                     : BR_WG_F128(0) : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));
    }
};
template <int TB> struct WgRS<16, TB> {                 // D[64 x 16] (+)= A[64 x 16] (registers) . B[16 x 16] (shared memory)
    static __device__ __forceinline__ void run(float (&d)[8], const uint32_t (&a)[4], uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, %14;\n}\n"
                     : BR_WG_F8(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate), "n"(TB));
    }
};
template <int TB> struct WgRS<32, TB> {                 // D[64 x 32] (+)= A[64 x 16] (registers) . B[16 x 32] (shared memory)
    static __device__ __forceinline__ void run(float (&d)[16], const uint32_t (&a)[4], uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, %22;\n}\n"
                     : BR_WG_F16(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate), "n"(TB));
    }
};
template <int TB> struct WgRS<64, TB> {                // D[64 x 64] (+)= A[64 x 16] (registers) . B[16 x 64] (shared memory)
    static __device__ __forceinline__ void run(float (&d)[32], const uint32_t (&a)[4], uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n}\n"
                     : BR_WG_F32(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate), "n"(TB));
    }
};
template <int TB> struct WgRS<128, TB> {                 // D[64 x 128] (+)= A[64 x 16] (registers) . B[16 x 128] (shared memory)
    static __device__ __forceinline__ void run(float (&d)[64], const uint32_t (&a)[4], uint64_t b, int accumulate) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, %70;\n}\n"
                     : BR_WG_F64(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate), "n"(TB));
    }
};
#undef BR_WG_F8
#undef BR_WG_F16
#undef BR_WG_F32
#undef BR_WG_F64
#undef BR_WG_F128

template <int N, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a, uint64_t b, int accumulate) { WgSS<N, TA, TB>::run(d, a, b, accumulate); }
template <int N, int TB = 0>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b, int accumulate) { WgRS<N, TB>::run(d, a, b, accumulate); }

}  // namespace br
