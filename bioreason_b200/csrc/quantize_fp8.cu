// Weight-only FP8 for the rollout decode: W [N, K] bf16 -> e4m3 codes in the decode GEMM's fragment-order layout (fp8_weights.cuh)
// plus one fp32 scale per output row.
//   scale[n] = amax_k |W[n, k]| / 448   (1 for an all-zero row)
//   Q[n, k]  = e4m3fn(W[n, k] / scale[n]), round to nearest even
// Both divisions are correctly rounded fp32 divisions, so the codes equal torch's (W.float() / scale[:, None]).to(float8_e4m3fn)
// bit for bit; |W / scale| <= 448 (up to the rounding of the division, which rounds back to 448), so no NaN code is produced.
#include <cuda_fp8.h>
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "fp8_weights.cuh"

namespace {

// one warp per row
__global__ void __launch_bounds__(256) row_scale_kernel(const bf16* __restrict__ W, long long ldw, int N, int K, float* __restrict__ scale) {
    const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= N) return;
    const bf16* row = W + (long long)n * ldw;
    float m = 0.f;
    for (int k = lane; k < K; k += 32) m = fmaxf(m, fabsf(__bfloat162float(row[k])));
    m = br::warp_max(m);
    if (lane == 0) scale[n] = m > 0.f ? __fdiv_rn(m, 448.f) : 1.f;
}

// one thread per 16 bytes of Q (one consumer thread's k16 slice of a unit)
__global__ void __launch_bounds__(256) quantize_kernel(const bf16* __restrict__ W, long long ldw, int N, int K, int KB,
                                                       const float* __restrict__ scale, uint4* __restrict__ Q, long long n_vec) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_vec) return;
    const long long u = i / (br::fp8w::UNIT_BYTES / 16);
    const int b0 = (int)(i - u * (br::fp8w::UNIT_BYTES / 16)) * 16;
    const int tile = (int)(u / KB), kb = (int)(u - (long long)tile * KB);
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        uint32_t word = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            int row, col;
            br::fp8w::unit_coord(b0 + 4 * j + c, row, col);
            const int n = tile * br::fp8w::UNIT_ROWS + row, k = kb * br::fp8w::UNIT_COLS + col;
            uint32_t code = 0;
            if (n < N && k < K) {
                const float x = __fdiv_rn(__bfloat162float(W[(long long)n * ldw + k]), scale[n]);
                code = (uint32_t)__nv_cvt_float_to_fp8(x, __NV_SATFINITE, __NV_E4M3);
            }
            word |= code << (8 * c);
        }
        w[j] = word;
    }
    Q[i] = make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace

extern "C" {

int64_t br_fp8_weight_bytes(int N, int K) { return N > 0 && K > 0 ? br::fp8w::bytes(N, K) : 0; }

int br_quantize_rows_e4m3(const void* W, int64_t ldw, int N, int K, void* Q, float* scale, void* stream) {
    BR_CHECK_ARG(N >= 1 && K >= 16 && K % 16 == 0 && ldw >= K, "quantize_rows_e4m3: need N >= 1, K a multiple of 16, ldw >= K (N=%d K=%d ldw=%lld)",
                 N, K, (long long)ldw);
    BR_CHECK_ARG(W && Q && scale, "quantize_rows_e4m3: W, Q and scale are required");
    BR_CHECK_ARG(((uintptr_t)Q & 15) == 0, "quantize_rows_e4m3: Q must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    row_scale_kernel<<<(N + 7) / 8, 256, 0, st>>>((const bf16*)W, ldw, N, K, scale);
    BR_CHECK_LAUNCH();
    const int KB = (K + br::fp8w::UNIT_COLS - 1) / br::fp8w::UNIT_COLS;
    const long long n_vec = br::fp8w::bytes(N, K) / 16;
    quantize_kernel<<<(unsigned)((n_vec + 255) / 256), 256, 0, st>>>((const bf16*)W, ldw, N, K, KB, scale, (uint4*)Q, n_vec);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // extern "C"
