// Flash attention backward on wgmma / TMA (sm_90a; causal GQA decoder rows, head_dim 128) -- autograd counterpart of
// attn_fwd_tc5.cu (SURVEY.md §2.3 K12).  Probabilities are recomputed from Q, K and the saved log-sum-exp; no score matrix, no
// fp32 atomics and no dQ workspace ever touch HBM, and every output element is produced by exactly one CTA in a fixed order, so
// the gradients are bit-reproducible run to run.
//
// Two kernels, one warpgroup per CTA, everything element-wise in registers (a quad of lanes shares a row of the tile):
//   dq kernel   : CTA = 64-query tile of one (row, query head); loops over the 64-key tiles it can see.
//                   S  = Q K^T,  dP = dO V^T                  (wgmma, both operands K-major in shared memory)
//                   dS = P o (dP - delta) * scale
//                   dQ += dS K                               (dS as the register A operand, the K tile as it landed, MN-major)
//                 also computes delta = rowsum(dO o O) for its rows and publishes it for the dk/dv kernel.
//   dk/dv kernel: CTA = 64-key tile of one (row, kv head); loops over the query heads of the group and the 64-query tiles that
//                 can see the keys; dK and dV accumulate in registers for the whole loop.
//                   S^T = K Q^T,  dP^T = V dO^T
//                   dV += P^T dO,  dK += dS^T Q               (P^T / dS^T as register A operands; dO and Q tiles MN-major)
// Thread 0 streams the per-iteration tiles through a two-stage TMA ring.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "wgmma.cuh"

namespace {

constexpr int D = 128, BT = 64, NTHREADS = 128;
constexpr int BLK = 64 * 128;             // bytes of a [64 rows x 64 cols] swizzled block
constexpr int TILE = 2 * BLK;             // a 64 x 128 bf16 tile
constexpr int OFF_R0 = 0, OFF_R1 = TILE, OFF_S0 = 2 * TILE, OFF_S1 = OFF_S0 + 2 * TILE, OFF_VEC = OFF_S1 + 2 * TILE, OFF_BAR = OFF_VEC + 2 * 64 * 4;
constexpr int SMEM = OFF_BAR + 64 + 1024; // two resident tiles + two streamed tiles x 2 stages
constexpr float LOG2E = 1.4426950408889634f;

struct BwdParams {
    const bf16 *o, *dout; long long ldo, lddo;
    const float* lse;        // [B, Hq, L]
    float* delta;            // [B, Hq, L]  (written by the dq kernel, read by the dk/dv kernel)
    bf16 *dq, *dk, *dv; long long lddq, lddk, lddv;
    int B, L, Hq, Hkv;
    const int *kv_start, *kv_end;
    float scale, scale_log2;
};

__device__ __forceinline__ float ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// acc[64 x 64] = A . B^T over d = 128, A and B K-major [64 x 128] tiles
__device__ __forceinline__ void mma_ss(float (&acc)[32], uint32_t a_addr, uint32_t b_addr) {
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t off = (kk >> 2) * BLK + (kk & 3) * 32;
        br::wgmma_ss<64>(acc, br::wg_desc_k(a_addr + off), br::wg_desc_k(b_addr + off), kk != 0);
    }
}
// acc[64 x 128] += A(registers: 64 x 64 bf16 from the fragment f) . B, B = a [64 (K) x 128 (N)] row-major tile (MN-major)
__device__ __forceinline__ void mma_rs(float (&acc)[64], const float (&f)[32], uint32_t b_addr) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a[4] = {br::pack_bf16(f[8 * kk + 0], f[8 * kk + 1]), br::pack_bf16(f[8 * kk + 2], f[8 * kk + 3]),
                               br::pack_bf16(f[8 * kk + 4], f[8 * kk + 5]), br::pack_bf16(f[8 * kk + 6], f[8 * kk + 7])};
        br::wgmma_rs<128, 1>(acc, a, br::wg_desc_mn(b_addr + kk * 2048, BLK, 1024), 1);
    }
}
__device__ __forceinline__ void tma_tile(uint8_t* dst, const CUtensorMap* tm, uint64_t* bar, int col0, int row0) {
    br::tma_load_2d(dst, tm, bar, col0, row0);
    br::tma_load_2d(dst + BLK, tm, bar, col0 + 64, row0);
}
// rows r0 and r0 + 8 of a [64 x 128] fragment -> bf16 rows (zero when `zero`)
__device__ __forceinline__ void store_frag(bf16* base, long long ld, int row0, int n_rows, const float (&acc)[64], int r0, int cq) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int r = row0 + r0 + 8 * hh;
        if (r >= n_rows) continue;
        bf16* dst = base + (long long)r * ld;
#pragma unroll
        for (int i = 0; i < 16; ++i) *reinterpret_cast<uint32_t*>(dst + 8 * i + cq) = br::pack_bf16(acc[4 * i + 2 * hh], acc[4 * i + 2 * hh + 1]);
    }
}

// =====================================================================================================================
// dq kernel
// =====================================================================================================================
__global__ void __launch_bounds__(NTHREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                   const __grid_constant__ CUtensorMap tmDO, const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* s_red = reinterpret_cast<float*>(smem + OFF_VEC);              // [2][64] delta halves
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* qdo_full = bars;                    // 1
    uint64_t* kv_full = bars + 1;                 // 2

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int qb = gridDim.x - 1 - blockIdx.x;
    const int h = blockIdx.y, b = blockIdx.z;
    const int hk = h / (p.Hq / p.Hkv);
    const int q0 = qb * BT;
    const int ks = p.kv_start ? p.kv_start[b] : 0;
    const int ke = p.kv_end ? p.kv_end[b] : p.L;
    const int last_key = min(ke - 1, q0 + BT - 1);
    const int jb_lo = ks / BT;
    int jb_hi = last_key >= 0 ? last_key / BT : -1;
    if (ke <= ks) jb_hi = jb_lo - 1;
    const int n_tiles = max(0, jb_hi - jb_lo + 1);

    auto load_kv = [&](int t) {
        const int st = t & 1, row_k = b * p.L + (jb_lo + t) * BT;
        br::mbar_expect_tx(&kv_full[st], 2 * TILE);
        tma_tile(smem + OFF_S0 + st * TILE, &tmK, &kv_full[st], hk * D, row_k);
        tma_tile(smem + OFF_S1 + st * TILE, &tmV, &kv_full[st], hk * D, row_k);
    };
    if (tid == 0) {
        br::tma_prefetch_desc(&tmQ); br::tma_prefetch_desc(&tmK); br::tma_prefetch_desc(&tmV); br::tma_prefetch_desc(&tmDO);
        br::mbar_init(qdo_full, 1); br::mbar_init(&kv_full[0], 1); br::mbar_init(&kv_full[1], 1);
        br::mbar_fence_init();
        if (n_tiles > 0) {
            const int row_q = b * p.L + q0;
            br::mbar_expect_tx(qdo_full, 2 * TILE);
            tma_tile(smem + OFF_R0, &tmQ, qdo_full, h * D, row_q);
            tma_tile(smem + OFF_R1, &tmDO, qdo_full, h * D, row_q);
            load_kv(0);
            if (n_tiles > 1) load_kv(1);
        }
    }
    // ---- delta = rowsum(dO o O) (fp32; two threads per query row, each half of the head dim, summed in a fixed order)
    {
        const int row = tid >> 1, half = tid & 1;
        const int i_glob = q0 + row;
        float delta = 0.f;
        if (i_glob < p.L) {
            const long long tok = (long long)b * p.L + i_glob;
            const uint4* op = reinterpret_cast<const uint4*>(p.o + tok * p.ldo + (long long)h * D + half * 64);
            const uint4* dp = reinterpret_cast<const uint4*>(p.dout + tok * p.lddo + (long long)h * D + half * 64);
            uint4 av[8], gv[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) { av[c] = __ldg(op + c); gv[c] = __ldg(dp + c); }
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 a = av[c], gd = gv[c];
                const float2 a0 = br::unpack_bf16(a.x), a1 = br::unpack_bf16(a.y), a2 = br::unpack_bf16(a.z), a3 = br::unpack_bf16(a.w);
                const float2 g0 = br::unpack_bf16(gd.x), g1 = br::unpack_bf16(gd.y), g2 = br::unpack_bf16(gd.z), g3 = br::unpack_bf16(gd.w);
                delta += a0.x * g0.x + a0.y * g0.y + a1.x * g1.x + a1.y * g1.y + a2.x * g2.x + a2.y * g2.y + a3.x * g3.x + a3.y * g3.y;
            }
        }
        s_red[half * 64 + row] = delta;
    }
    __syncthreads();
    if (tid < 64 && q0 + tid < p.L) p.delta[((long long)b * p.Hq + h) * p.L + q0 + tid] = s_red[tid] + s_red[64 + tid];
    const int r0 = warp * 16 + (lane >> 2), cq = 2 * (lane & 3);
    float lse2[2], delta_s[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int i_glob = q0 + r0 + 8 * hh;
        lse2[hh] = i_glob < p.L ? p.lse[((long long)b * p.Hq + h) * p.L + i_glob] * LOG2E : INFINITY;
        delta_s[hh] = (s_red[r0 + 8 * hh] + s_red[64 + r0 + 8 * hh]) * p.scale;    // same fixed order as the published value
    }
    float dq[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) dq[i] = 0.f;
    const uint32_t q_addr = br::smem_u32(smem + OFF_R0), do_addr = br::smem_u32(smem + OFF_R1);
    if (n_tiles > 0) br::mbar_wait(qdo_full, 0);
    for (int t = 0; t < n_tiles; ++t) {
        const int st = t & 1;
        const int k0 = (jb_lo + t) * BT;
        const uint32_t k_addr = br::smem_u32(smem + OFF_S0 + st * TILE), v_addr = br::smem_u32(smem + OFF_S1 + st * TILE);
        br::mbar_wait(&kv_full[st], (t >> 1) & 1);
        float s[32], dp[32];
        br::wg_fence();
        mma_ss(s, q_addr, k_addr);                                            // S = Q K^T
        mma_ss(dp, do_addr, v_addr);                                          // dP = dO V^T
        br::wg_commit();
        br::wg_wait<0>();
        br::wg_fence_operand(s);
        br::wg_fence_operand(dp);
        const bool need_mask = (k0 < ks) || (k0 + BT > ke) || (k0 + BT - 1 > q0);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int x = 4 * i + 2 * hh + e;
                    const int j = k0 + 8 * i + cq + e, ig = q0 + r0 + 8 * hh;
                    float sv = s[x];
                    if (need_mask && !((j >= ks) && (j < ke) && (j <= ig))) sv = -INFINITY;      // -inf score -> probability 0
                    const float pr = ex2(fmaf(sv, p.scale_log2, -lse2[hh]));
                    s[x] = pr * fmaf(dp[x], p.scale, -delta_s[hh]);                              // dS
                }
        br::wg_fence();
        mma_rs(dq, s, k_addr);                                                // dQ += dS K
        br::wg_commit();
        br::wg_wait<0>();
        br::wg_fence_operand(dq);
        __syncthreads();
        if (tid == 0 && t + 2 < n_tiles) load_kv(t + 2);
    }
    store_frag(p.dq + (long long)b * p.L * p.lddq + (long long)h * D, p.lddq, q0, p.L, dq, r0, cq);
}

// =====================================================================================================================
// dk / dv kernel
// =====================================================================================================================
__global__ void __launch_bounds__(NTHREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmDO, const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* kv_full = bars;                     // 1
    uint64_t* qdo_full = bars + 1;                // 2

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int jb = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
    const int GQ = p.Hq / p.Hkv;
    const int key0 = jb * BT;
    const int ks = p.kv_start ? p.kv_start[b] : 0;
    const int ke = p.kv_end ? p.kv_end[b] : p.L;
    const bool block_live = (key0 < ke) && (key0 + BT > ks) && (key0 < p.L);
    const int n_ib = (p.L + BT - 1) / BT;                                 // 64-query tiles
    const int ib_lo = key0 / BT;                                          // causal: the first query tile that sees a key of this block
    const int per_head = n_ib - ib_lo;
    const int iters = block_live ? GQ * per_head : 0;

    auto load_qdo = [&](int it) {
        const int st = it & 1;
        const int h = hk * GQ + it / per_head, ib = ib_lo + it % per_head;
        const int row_q = b * p.L + ib * BT;
        br::mbar_expect_tx(&qdo_full[st], 2 * TILE);
        tma_tile(smem + OFF_S0 + st * TILE, &tmQ, &qdo_full[st], h * D, row_q);
        tma_tile(smem + OFF_S1 + st * TILE, &tmDO, &qdo_full[st], h * D, row_q);
    };
    if (tid == 0) {
        br::tma_prefetch_desc(&tmQ); br::tma_prefetch_desc(&tmK); br::tma_prefetch_desc(&tmV); br::tma_prefetch_desc(&tmDO);
        br::mbar_init(kv_full, 1); br::mbar_init(&qdo_full[0], 1); br::mbar_init(&qdo_full[1], 1);
        br::mbar_fence_init();
        if (iters > 0) {
            const int row_k = b * p.L + key0;
            br::mbar_expect_tx(kv_full, 2 * TILE);
            tma_tile(smem + OFF_R0, &tmK, kv_full, hk * D, row_k);
            tma_tile(smem + OFF_R1, &tmV, kv_full, hk * D, row_k);
            load_qdo(0);
            if (iters > 1) load_qdo(1);
        }
    }
    __syncthreads();
    const int r0 = warp * 16 + (lane >> 2), cq = 2 * (lane & 3);
    bool key_ok[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) { const int j = key0 + r0 + 8 * hh; key_ok[hh] = (j >= ks) && (j < ke); }
    float dk[64], dv[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
    const uint32_t k_addr = br::smem_u32(smem + OFF_R0), v_addr = br::smem_u32(smem + OFF_R1);
    if (iters > 0) br::mbar_wait(kv_full, 0);
    for (int it = 0; it < iters; ++it) {
        const int st = it & 1;
        const int h = hk * GQ + it / per_head, ib = ib_lo + it % per_head;
        const int q0 = ib * BT;
        // per-query vectors of this thread's 16 columns (queries beyond L carry lse = +inf: probability 0)
        float l2[16], dd[16];
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            const int i = q0 + 8 * (c >> 1) + cq + (c & 1);
            const long long off = ((long long)b * p.Hq + h) * p.L + i;
            l2[c] = i < p.L ? __ldg(p.lse + off) * LOG2E : INFINITY;
            dd[c] = i < p.L ? __ldcg(p.delta + off) * p.scale : 0.f;
        }
        const uint32_t q_addr = br::smem_u32(smem + OFF_S0 + st * TILE), do_addr = br::smem_u32(smem + OFF_S1 + st * TILE);
        br::mbar_wait(&qdo_full[st], (it >> 1) & 1);
        float s[32], dp[32];
        br::wg_fence();
        mma_ss(s, k_addr, q_addr);                                            // S^T = K Q^T
        mma_ss(dp, v_addr, do_addr);                                          // dP^T = V dO^T
        br::wg_commit();
        br::wg_wait<0>();
        br::wg_fence_operand(s);
        br::wg_fence_operand(dp);
        const bool need_mask = (q0 < key0 + BT - 1) || (key0 < ks) || (key0 + BT > ke);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int x = 4 * i + 2 * hh + e, c = 2 * i + e;
                    const int qi = q0 + 8 * i + cq + e, j = key0 + r0 + 8 * hh;
                    float sv = s[x];
                    if (need_mask && !(key_ok[hh] && j <= qi)) sv = -INFINITY;
                    const float pr = ex2(fmaf(sv, p.scale_log2, -l2[c]));
                    s[x] = pr;                                                                   // P^T
                    dp[x] = pr * fmaf(dp[x], p.scale, -dd[c]);                                   // dS^T
                }
        br::wg_fence();
        mma_rs(dv, s, do_addr);                                               // dV += P^T dO
        mma_rs(dk, dp, q_addr);                                               // dK += dS^T Q
        br::wg_commit();
        br::wg_wait<0>();
        br::wg_fence_operand(dv);
        br::wg_fence_operand(dk);
        __syncthreads();
        if (tid == 0 && it + 2 < iters) load_qdo(it + 2);
    }
    store_frag(p.dk + (long long)b * p.L * p.lddk + (long long)hk * D, p.lddk, key0, p.L, dk, r0, cq);
    store_frag(p.dv + (long long)b * p.L * p.lddv + (long long)hk * D, p.lddv, key0, p.L, dv, r0, cq);
}

}  // namespace

int br_attn_bwd_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                         const void* dout, int64_t lddo, const float* lse, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv,
                         int B, int L, int n_q_heads, int n_kv_heads, const int32_t* kv_start, const int32_t* kv_end, float scale,
                         void* workspace, cudaStream_t st) {
    BwdParams p;
    p.o = (const bf16*)o; p.dout = (const bf16*)dout; p.ldo = ldo; p.lddo = lddo; p.lse = lse; p.delta = (float*)workspace;
    p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv; p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
    p.B = B; p.L = L; p.Hq = n_q_heads; p.Hkv = n_kv_heads; p.kv_start = kv_start; p.kv_end = kv_end;
    p.scale = scale; p.scale_log2 = scale * LOG2E;
    BR_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 && lddk % 8 == 0 && lddv % 8 == 0,
                 "attn_bwd: strides must be multiples of 8 elements");
    BR_CHECK_ARG(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)o | (uintptr_t)dout | (uintptr_t)dq | (uintptr_t)dk | (uintptr_t)dv) % 16 == 0,
                 "attn_bwd: tensors must be 16-byte aligned");
    CUtensorMap tq, tk, tv, tdo;                                     // 64-row boxes
    int rc;
    const uint64_t rows = (uint64_t)B * L;
    if ((rc = br_make_tmap_2d_bf16(&tq, q, rows, (uint64_t)n_q_heads * D, ldq, BT))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tk, k, rows, (uint64_t)n_kv_heads * D, ldk, BT))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tv, v, rows, (uint64_t)n_kv_heads * D, ldv, BT))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tdo, dout, rows, (uint64_t)n_q_heads * D, lddo, BT))) return rc;
    static bool done = false;
    if (!done) {
        BR_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        BR_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        done = true;
    }
    const int nb = (L + BT - 1) / BT;
    attn_bwd_dq_kernel<<<dim3(nb, n_q_heads, B), NTHREADS, SMEM, st>>>(tq, tk, tv, tdo, p);
    BR_CHECK_LAUNCH();
    attn_bwd_dkv_kernel<<<dim3(nb, n_kv_heads, B), NTHREADS, SMEM, st>>>(tq, tk, tv, tdo, p);
    BR_CHECK_LAUNCH();
    return BR_OK;
}
