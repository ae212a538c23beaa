// LoRA down-projection with dropout on wgmma (sm_90a):  t[M, n_proj * r] = scale * inv_keep * ((x . m_j) . A_j^T).
//
// peft computes every adapted projection as base(x) + s * B(A(dropout(x))) with its own dropout draw (reason.py:376-384); the fused
// q|k|v and gate|up linears share one input x but need one mask per projection.  The product is HBM-bound on x, so x is read once:
//   warp 4      TMA producer : [64 rows x 64 cols] tiles of x and the [n_proj * r x 64] tile of the stacked A, NSTAGE ring
//   warps 0..3  one consumer warpgroup (64 rows): ldmatrix the x fragment into registers, AND it with each projection's mask
//               (counter-based, lora_dropout.cuh), and issue the register-A wgmma into that projection's accumulator; the epilogue
//               scales by s / (1 - p_eff) and rounds to bf16 once, like the unmasked A-GEMM.
// The base GEMM (x . W^T + t . B^T) reads the undropped x and is unchanged.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "lora_dropout.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 64, BK = 64, NTHREADS = 160, NSTAGE = 4;
constexpr int X_BYTES = BM * BK * 2;

struct DownParams {
    int M, K;
    bf16* t; long long ldt;
    float alpha;
    br::DropParams d;
};

template <int R, int NP>
__global__ void __launch_bounds__(NTHREADS)
lora_down_dropout_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmA, const DownParams p) {
    constexpr int STAGE = X_BYTES + NP * R * 128;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE);
    uint64_t* empty_bar = full_bar + NSTAGE;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * BM;
    const int n_kb = (p.K + BK - 1) / BK;

    if (threadIdx.x == 0) {
        br::tma_prefetch_desc(&tmX); br::tma_prefetch_desc(&tmA);
        for (int s = 0; s < NSTAGE; ++s) { br::mbar_init(&full_bar[s], 1); br::mbar_init(&empty_bar[s], 1); }
        br::mbar_fence_init();
    }
    __syncthreads();

    if (warp == 4) {
        if (lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int kb = 0; kb < n_kb; ++kb) {
                br::mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* st = smem + s * STAGE;
                br::mbar_expect_tx(&full_bar[s], STAGE);
                br::tma_load_2d(st, &tmX, &full_bar[s], kb * BK, m0);
                br::tma_load_2d(st + X_BYTES, &tmA, &full_bar[s], kb * BK, 0);
                if (++s == NSTAGE) { s = 0; ph ^= 1; }
            }
        }
        return;
    }
    const int q = lane & 3;
    const int lrow = 16 * warp + (lane >> 2);                       // fragment rows lrow, lrow + 8 of the 64-row tile
    const long long grow = p.d.row0 + m0 + lrow;
    // ldmatrix.x4 address of this lane: matrices (rows 0-7 | 8-15) x (k 0-7 | 8-15) of the warp's 16-row slice; 128B swizzle
    const int ld_row = 16 * warp + (lane & 7) + (((lane >> 3) & 1) << 3);
    const int ld_hi = lane >> 4;
    float acc[NP][R / 2];
#pragma unroll
    for (int j = 0; j < NP; ++j)
#pragma unroll
        for (int i = 0; i < R / 2; ++i) acc[j][i] = 0.f;
    int s = 0; uint32_t ph = 0;
    for (int kb = 0; kb < n_kb; ++kb) {
        br::mbar_wait(&full_bar[s], ph);
        const uint32_t sx = br::smem_u32(smem + s * STAGE);
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
            uint32_t a[4];
            const int chunk = 2 * kk + ld_hi;
            br::ldsm_x4(a, sx + ld_row * 128 + ((chunk ^ (ld_row & 7)) << 4));
            // a[i]: row lrow + 8 (i & 1), columns 8 (cg0 + (i >> 1)) + 2q, +1; lane q draws group i = q of the quad
            const int cg0 = (kb * BK + kk * 16) >> 3;
            uint32_t am[NP][4];
#pragma unroll
            for (int j = 0; j < NP; ++j) {
                uint32_t w[4];
                br::quad_words(br::drop_group(p.d, grow + 8 * (q & 1), cg0 + (q >> 1), p.d.proj + j), w);
#pragma unroll
                for (int i = 0; i < 4; ++i) am[j][i] = a[i] & br::keep_bits(w[i], p.d.T);
            }
            br::wg_fence();
#pragma unroll
            for (int j = 0; j < NP; ++j)
                br::wgmma_rs<R>(acc[j], am[j], br::wg_desc_k(sx + X_BYTES + j * R * 128) + 2 * kk, 1);
        }
        br::wg_commit();
        br::wg_wait<0>();
#pragma unroll
        for (int j = 0; j < NP; ++j) br::wg_fence_operand(acc[j]);
        if (threadIdx.x == 0) br::mbar_arrive(&empty_bar[s]);
        if (++s == NSTAGE) { s = 0; ph ^= 1; }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int row = m0 + lrow + 8 * hh;
        if (row >= p.M) continue;
        bf16* out = p.t + (long long)row * p.ldt + 2 * q;
#pragma unroll
        for (int j = 0; j < NP; ++j)
#pragma unroll
            for (int i = 0; i < R / 8; ++i)
                *reinterpret_cast<uint32_t*>(out + j * R + 8 * i) =
                    br::pack_bf16(acc[j][4 * i + 2 * hh] * p.alpha, acc[j][4 * i + 2 * hh + 1] * p.alpha);
    }
}

template <int R, int NP>
int launch_down(const CUtensorMap& tx, const CUtensorMap& ta, const DownParams& p, cudaStream_t st) {
    constexpr int SMEM = NSTAGE * (X_BYTES + NP * R * 128) + 256 + 1024;
    auto kern = lora_down_dropout_kernel<R, NP>;
    static bool done = false;
    if (!done) { BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM)); done = true; }
    kern<<<(p.M + BM - 1) / BM, NTHREADS, SMEM, st>>>(tx, ta, p);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

template <int R>
int launch_down_np(int np, const CUtensorMap& tx, const CUtensorMap& ta, const DownParams& p, cudaStream_t st) {
    if (np == 1) return launch_down<R, 1>(tx, ta, p, st);
    if (np == 2) return launch_down<R, 2>(tx, ta, p, st);
    return launch_down<R, 3>(tx, ta, p, st);
}

__global__ void dropout_mask_kernel(const br::DropParams d, int M, int K, uint8_t* __restrict__ keep, long long ldo) {
    const int ng = (K + 7) >> 3;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)M * ng) return;
    const int m = (int)(g / ng), cg = (int)(g % ng);
    const uint4 w = br::drop_group(d, d.row0 + m, cg, d.proj);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int col = 8 * cg + e;
        if (col < K) keep[(long long)m * ldo + col] = ((br::sel4(w, e >> 1) >> (16 * (e & 1))) & 0xFFFFu) >= (uint32_t)d.T ? 1 : 0;
    }
}

}  // namespace

extern "C" {

int br_lora_down_dropout(const void* x, int64_t ldx, const void* A, int64_t lda, void* t, int64_t ldt, int M, int K, int n_proj,
                         float scale, const br_lora_dropout* d, void* stream) {
    int rc;
    if ((rc = br::check_drop(d, "lora_down_dropout"))) return rc;
    const int r = d->r;
    BR_CHECK_ARG(M > 0 && K > 0 && K % 8 == 0 && ldx % 8 == 0 && lda % 8 == 0 && ldt % 2 == 0, "lora_down_dropout: M=%d K=%d (K, ld %% 8)", M, K);
    BR_CHECK_ARG(n_proj >= 1 && n_proj <= 3, "lora_down_dropout: n_proj=%d outside [1, 3]", n_proj);
    BR_CHECK_ARG(r == 16 || r == 32 || r == 64, "lora_down_dropout: rank %d not in {16, 32, 64}", r);
    BR_CHECK_ARG(((uintptr_t)x % 16 == 0) && ((uintptr_t)A % 16 == 0) && ((uintptr_t)t % 4 == 0), "lora_down_dropout: alignment");
    DownParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.K = K; p.t = reinterpret_cast<bf16*>(t); p.ldt = ldt;
    p.d = br::drop_params(*d);
    p.alpha = scale * d->inv_keep;
    CUtensorMap tx, ta;
    if ((rc = br_make_tmap_2d_bf16(&tx, x, (uint64_t)M, (uint64_t)K, (uint64_t)ldx, BM))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&ta, A, (uint64_t)(n_proj * r), (uint64_t)K, (uint64_t)lda, n_proj * r))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (r == 16) return launch_down_np<16>(n_proj, tx, ta, p, st);
    if (r == 32) return launch_down_np<32>(n_proj, tx, ta, p, st);
    return launch_down_np<64>(n_proj, tx, ta, p, st);
}

int br_lora_dropout_mask(const br_lora_dropout* d, int M, int K, uint8_t* keep, int64_t ldo, void* stream) {
    int rc;
    if ((rc = br::check_drop(d, "lora_dropout_mask"))) return rc;
    BR_CHECK_ARG(M > 0 && K > 0 && ldo >= K && keep, "lora_dropout_mask: M=%d K=%d ldo=%lld", M, K, (long long)ldo);
    const long long n = (long long)M * ((K + 7) / 8);
    dropout_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(br::drop_params(*d), M, K, keep, ldo);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // extern "C"
