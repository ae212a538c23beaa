// FP8 (e4m3) decode weights: the byte layout shared by br_quantize_rows_e4m3 (producer) and the FP8 instantiation of the decode
// GEMM (consumer).  Nothing outside these two kernels knows it: Python holds an opaque byte buffer plus one fp32 scale per row.
//
// A matrix W [N, K] is cut into units of 128 rows x 64 columns, unit u = tile * KB + kb (KB = ceil(K / 64)), 8192 bytes each, stored
// back to back (a stream-K chunk of consecutive units is one contiguous byte range; rows >= N and columns >= K hold zero codes).
// Inside a unit the bytes are in register-A fragment order of the m64n*k16 wgmma: for k16 slice ks, consumer thread t (0..127),
// A register j (0..3), element e (low / high half of the bf16 pair) and m64 half h,
//     byte ks * 2048 + t * 16 + j * 4 + e * 2 + h
//   = code of W[128 tile + 64 h + 16 (t / 32) + (t % 32) / 4 + 8 (j & 1),  64 kb + 16 ks + 2 (t % 4) + 8 (j >> 1) + e]
// so a unit is fetched with one bulk copy and each thread reads its 16 bytes of a k16 slice (both m64 halves) with one conflict-free
// 16-byte shared load, without swizzle.
#pragma once
#include <stdint.h>

namespace br {
namespace fp8w {

constexpr int UNIT_ROWS = 128, UNIT_COLS = 64, UNIT_BYTES = UNIT_ROWS * UNIT_COLS;

__host__ __device__ __forceinline__ int64_t bytes(int N, int K) {
    return (int64_t)((N + UNIT_ROWS - 1) / UNIT_ROWS) * ((K + UNIT_COLS - 1) / UNIT_COLS) * UNIT_BYTES;
}

// (row, column) within its unit of byte `b` of the unit (0 <= b < UNIT_BYTES)
__host__ __device__ __forceinline__ void unit_coord(int b, int& row, int& col) {
    const int ks = b >> 11, t = (b >> 4) & 127, j = (b >> 2) & 3, e = (b >> 1) & 1, h = b & 1;
    row = 64 * h + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * (j & 1);
    col = 16 * ks + 2 * (t & 3) + 8 * (j >> 1) + e;
}

#ifdef __CUDACC__
// One 32-bit word of the layout (bytes: e0 h0 | e0 h1 | e1 h0 | e1 h1) -> the bf16x2 A registers of both m64 halves, exactly.
// The sign and the 7 exponent/mantissa bits of each code are placed where bf16 keeps them, which reads the code as a bf16 whose
// value is the e4m3 value times 2^-120 (normal and subnormal codes alike); one bf16 multiply by 2^120 (exact: a power of two,
// bf16 arithmetic keeps subnormal inputs) gives the value.
__device__ __forceinline__ void e4m3x4_to_bf16x2(uint32_t q, uint32_t& h0, uint32_t& h1) {
    const uint32_t x0 = q << 8;
    const uint32_t b0 = (x0 & 0x80008000u) | ((x0 & 0x7F007F00u) >> 4);
    const uint32_t b1 = (q & 0x80008000u) | ((q & 0x7F007F00u) >> 4);
    const uint32_t two120 = 0x7B807B80u;                                   // bf16x2 (2^120, 2^120)
    asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(h0) : "r"(b0), "r"(two120));
    asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(h1) : "r"(b1), "r"(two120));
}
#endif

}  // namespace fp8w
}  // namespace br
