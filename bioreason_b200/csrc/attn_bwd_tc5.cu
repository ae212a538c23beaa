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
//
// Shared-prefix layout (br_attn_bwd_shared): the buffer holds U groups of G rows as [U * Lp prefix rows | R = U * G suffixes of Ls rows],
// Lp a multiple of 64 (see br_attn_fwd_shared).  Four launches, each output element still written by one CTA in a fixed order:
//   prefix dQ      : the dense dq kernel on [U, Lp];
//   suffix dQ      : the dq kernel in SHARED mode (key tiles j < Lp / 64 from the group's prefix rows, the rest from the row's suffix);
//   suffix dK / dV : the dense dk/dv kernel on [R, Ls] with the windows shifted by Lp (suffix keys are seen by their own row only);
//   prefix dK / dV : the dk/dv kernel in PREFIX mode: per query head, the group's prefix query tiles, then every query tile of suffix rows
//                    g = 0 .. G-1 (with G = 1 this is the dense kernel's order, so the result equals the dense one bit for bit).
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
    // shared-prefix modes: kv_start per group; suffix lse / delta [R, Hq, Ls] (the prefix ones are lse / delta above, [U, Hq, Lp])
    int G, Lp, Ls;
    long long sfx0;          // first suffix row of the buffer (U * Lp)
    const float* lse_s;
    float* delta_s;
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
template <bool SHARED>
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
    const int qb = (SHARED ? p.Lp / BT : 0) + gridDim.x - 1 - blockIdx.x;
    const int h = blockIdx.y, b = blockIdx.z;
    const int hk = h / (p.Hq / p.Hkv);
    const int q0 = qb * BT;
    const int ks = p.kv_start ? p.kv_start[SHARED ? b / p.G : b] : 0;
    const int ke = p.kv_end ? p.kv_end[b] : p.L;
    const int last_key = min(ke - 1, q0 + BT - 1);
    // shared mode: buffer row of position i (>= Lp) of this CTA's row, and index of (b, h, i) in the suffix lse / delta
    auto tok_row = [&](int i) -> long long { return SHARED ? p.sfx0 + (long long)b * p.Ls + (i - p.Lp) : (long long)b * p.L + i; };
    auto vec_idx = [&](int i) -> long long { return ((long long)b * p.Hq + h) * p.Ls + i - p.Lp; };
    const int jb_lo = ks / BT;
    int jb_hi = last_key >= 0 ? last_key / BT : -1;
    if (ke <= ks) jb_hi = jb_lo - 1;
    const int n_tiles = max(0, jb_hi - jb_lo + 1);

    auto load_kv = [&](int t) {
        const int st = t & 1, j0 = (jb_lo + t) * BT;
        const int row_k = SHARED ? (j0 < p.Lp ? (b / p.G) * p.Lp + j0 : (int)tok_row(j0)) : b * p.L + (jb_lo + t) * BT;
        br::mbar_expect_tx(&kv_full[st], 2 * TILE);
        tma_tile(smem + OFF_S0 + st * TILE, &tmK, &kv_full[st], hk * D, row_k);
        tma_tile(smem + OFF_S1 + st * TILE, &tmV, &kv_full[st], hk * D, row_k);
    };
    if (tid == 0) {
        br::tma_prefetch_desc(&tmQ); br::tma_prefetch_desc(&tmK); br::tma_prefetch_desc(&tmV); br::tma_prefetch_desc(&tmDO);
        br::mbar_init(qdo_full, 1); br::mbar_init(&kv_full[0], 1); br::mbar_init(&kv_full[1], 1);
        br::mbar_fence_init();
        if (n_tiles > 0) {
            const int row_q = SHARED ? (int)tok_row(q0) : b * p.L + q0;
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
            const long long tok = tok_row(i_glob);
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
    if (tid < 64 && q0 + tid < p.L) {
        if constexpr (SHARED) p.delta_s[vec_idx(q0 + tid)] = s_red[tid] + s_red[64 + tid];
        else p.delta[((long long)b * p.Hq + h) * p.L + q0 + tid] = s_red[tid] + s_red[64 + tid];
    }
    const int r0 = warp * 16 + (lane >> 2), cq = 2 * (lane & 3);
    float lse2[2], delta_s[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int i_glob = q0 + r0 + 8 * hh;
        if constexpr (SHARED) lse2[hh] = i_glob < p.L ? p.lse_s[vec_idx(i_glob)] * LOG2E : INFINITY;
        else lse2[hh] = i_glob < p.L ? p.lse[((long long)b * p.Hq + h) * p.L + i_glob] * LOG2E : INFINITY;
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
    bf16* dq_base = SHARED ? p.dq + tok_row(0) * p.lddq : p.dq + (long long)b * p.L * p.lddq;   // row 0 of b (never addressed when SHARED)
    store_frag(dq_base + (long long)h * D, p.lddq, q0, p.L, dq, r0, cq);
}

// =====================================================================================================================
// dk / dv kernel
// =====================================================================================================================
template <bool PREFIX>
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
    const int n_sb = PREFIX ? (p.Ls + BT - 1) / BT : 1;                   // PREFIX: query tiles of one suffix
    const int per_head = n_ib - ib_lo + (PREFIX ? p.G * n_sb : 0);
    const int iters = block_live ? GQ * per_head : 0;
    // query tile k (0 <= k < per_head) of head h: buffer row and position of its first query, index of that query in its lse / delta
    // vectors, and the number of valid queries
    struct QTile { long long row, vrow; int q0, n_valid; const float* lse; const float* delta; };
    auto qtile = [&](int k, int h) -> QTile {
        QTile t;
        if (!PREFIX || k < n_ib - ib_lo) {
            const int ib = ib_lo + k;
            t.row = (long long)b * p.L + ib * BT; t.q0 = ib * BT; t.n_valid = p.L - ib * BT;
            t.vrow = ((long long)b * p.Hq + h) * p.L + ib * BT; t.lse = p.lse; t.delta = p.delta;
        } else {
            const int ks2 = k - (n_ib - ib_lo), g = ks2 / n_sb, sb = ks2 - g * n_sb;
            const long long r = (long long)b * p.G + g;
            t.row = p.sfx0 + r * p.Ls + sb * BT; t.q0 = p.L + sb * BT; t.n_valid = p.Ls - sb * BT;      // PREFIX: p.L = Lp
            t.vrow = (r * p.Hq + h) * p.Ls + sb * BT; t.lse = p.lse_s; t.delta = p.delta_s;
        }
        return t;
    };

    auto load_qdo = [&](int it) {
        const int st = it & 1;
        const int h = hk * GQ + it / per_head;
        const int row_q = PREFIX ? (int)qtile(it % per_head, h).row : b * p.L + (ib_lo + it % per_head) * BT;
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
        const int h = hk * GQ + it / per_head;
        int q0;
        // per-query vectors of this thread's 16 columns (queries beyond the row end carry lse = +inf: probability 0)
        float l2[16], dd[16];
        if constexpr (PREFIX) {
            const QTile qt = qtile(it % per_head, h);
            q0 = qt.q0;
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                const int i = 8 * (c >> 1) + cq + (c & 1);
                l2[c] = i < qt.n_valid ? __ldg(qt.lse + qt.vrow + i) * LOG2E : INFINITY;
                dd[c] = i < qt.n_valid ? __ldcg(qt.delta + qt.vrow + i) * p.scale : 0.f;
            }
        } else {
            const int ib = ib_lo + it % per_head;
            q0 = ib * BT;
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                const int i = q0 + 8 * (c >> 1) + cq + (c & 1);
                const long long off = ((long long)b * p.Hq + h) * p.L + i;
                l2[c] = i < p.L ? __ldg(p.lse + off) * LOG2E : INFINITY;
                dd[c] = i < p.L ? __ldcg(p.delta + off) * p.scale : 0.f;
            }
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

__global__ void shift_windows_kernel(const int* kv_start, const int* kv_end, int G, int R, int Lp, int* ks_s, int* ke_s) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    ks_s[r] = max(kv_start[r / G] - Lp, 0);
    ke_s[r] = max(kv_end[r] - Lp, 0);
}

int set_smem_once() {
    static bool done = false;
    if (!done) {
        BR_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        BR_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        BR_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        BR_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        done = true;
    }
    return BR_OK;
}

// q / k / v / dout tensor maps (64-row boxes) over `rows` buffer rows starting at row `row0`
int make_maps(CUtensorMap (&tm)[4], const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* dout,
              int64_t lddo, long long row0, uint64_t rows, int n_q_heads, int n_kv_heads) {
    int rc;
    if ((rc = br_make_tmap_2d_bf16(&tm[0], (const bf16*)q + row0 * ldq, rows, (uint64_t)n_q_heads * D, ldq, BT))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tm[1], (const bf16*)k + row0 * ldk, rows, (uint64_t)n_kv_heads * D, ldk, BT))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tm[2], (const bf16*)v + row0 * ldv, rows, (uint64_t)n_kv_heads * D, ldv, BT))) return rc;
    return br_make_tmap_2d_bf16(&tm[3], (const bf16*)dout + row0 * lddo, rows, (uint64_t)n_q_heads * D, lddo, BT);
}

}  // namespace

int br_attn_bwd_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                         const void* dout, int64_t lddo, const float* lse, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv,
                         int B, int L, int n_q_heads, int n_kv_heads, const int32_t* kv_start, const int32_t* kv_end, float scale,
                         void* workspace, cudaStream_t st) {
    BwdParams p = {};
    p.o = (const bf16*)o; p.dout = (const bf16*)dout; p.ldo = ldo; p.lddo = lddo; p.lse = lse; p.delta = (float*)workspace;
    p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv; p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
    p.B = B; p.L = L; p.Hq = n_q_heads; p.Hkv = n_kv_heads; p.kv_start = kv_start; p.kv_end = kv_end;
    p.scale = scale; p.scale_log2 = scale * LOG2E;
    BR_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 && lddk % 8 == 0 && lddv % 8 == 0,
                 "attn_bwd: strides must be multiples of 8 elements");
    BR_CHECK_ARG(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)o | (uintptr_t)dout | (uintptr_t)dq | (uintptr_t)dk | (uintptr_t)dv) % 16 == 0,
                 "attn_bwd: tensors must be 16-byte aligned");
    CUtensorMap tm[4];
    int rc;
    if ((rc = make_maps(tm, q, ldq, k, ldk, v, ldv, dout, lddo, 0, (uint64_t)B * L, n_q_heads, n_kv_heads))) return rc;
    if ((rc = set_smem_once())) return rc;
    const int nb = (L + BT - 1) / BT;
    attn_bwd_dq_kernel<false><<<dim3(nb, n_q_heads, B), NTHREADS, SMEM, st>>>(tm[0], tm[1], tm[2], tm[3], p);
    BR_CHECK_LAUNCH();
    attn_bwd_dkv_kernel<false><<<dim3(nb, n_kv_heads, B), NTHREADS, SMEM, st>>>(tm[0], tm[1], tm[2], tm[3], p);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int64_t br_attn_bwd_shared_workspace_bytes_impl(int U, int G, int Lp, int Ls, int n_q_heads) {
    const int64_t R = (int64_t)U * G;
    return ((int64_t)U * Lp + R * Ls) * n_q_heads * (int64_t)sizeof(float) + 2 * R * (int64_t)sizeof(int32_t);
}

int br_attn_bwd_shared_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o, int64_t ldo,
                                const void* dout, int64_t lddo, const float* lse_prefix, const float* lse_suffix, void* dq, int64_t lddq,
                                void* dk, int64_t lddk, void* dv, int64_t lddv, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads,
                                const int32_t* kv_start, const int32_t* kv_end, float scale, void* workspace, cudaStream_t st) {
    BR_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 && lddk % 8 == 0 && lddv % 8 == 0,
                 "attn_bwd_shared: strides must be multiples of 8 elements");
    BR_CHECK_ARG(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)o | (uintptr_t)dout | (uintptr_t)dq | (uintptr_t)dk | (uintptr_t)dv) % 16 == 0,
                 "attn_bwd_shared: tensors must be 16-byte aligned");
    const int R = U * G;
    const long long sfx0 = (long long)U * Lp;
    float* delta_p = (float*)workspace;
    float* delta_s = delta_p + sfx0 * n_q_heads;
    int* ks_s = (int*)(delta_s + (long long)R * Ls * n_q_heads);
    int* ke_s = ks_s + R;
    CUtensorMap tm[4], tm_s[4];                                      // whole buffer; suffix rows only
    int rc;
    if ((rc = make_maps(tm, q, ldq, k, ldk, v, ldv, dout, lddo, 0, (uint64_t)(sfx0 + (long long)R * Ls), n_q_heads, n_kv_heads))) return rc;
    if ((rc = make_maps(tm_s, q, ldq, k, ldk, v, ldv, dout, lddo, sfx0, (uint64_t)R * Ls, n_q_heads, n_kv_heads))) return rc;
    if ((rc = set_smem_once())) return rc;
    BwdParams p = {};
    p.o = (const bf16*)o; p.dout = (const bf16*)dout; p.ldo = ldo; p.lddo = lddo;
    p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv; p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
    p.Hq = n_q_heads; p.Hkv = n_kv_heads; p.scale = scale; p.scale_log2 = scale * LOG2E;
    p.G = G; p.Lp = Lp; p.Ls = Ls; p.sfx0 = sfx0; p.lse_s = lse_suffix; p.delta_s = delta_s;
    p.kv_start = kv_start;
    const int np = Lp / BT, ns = (Ls + BT - 1) / BT;
    // prefix dQ (+ prefix delta): dense kernel on [U, Lp]
    BwdParams pp = p;
    pp.B = U; pp.L = Lp; pp.lse = lse_prefix; pp.delta = delta_p; pp.kv_end = nullptr;
    if (np > 0) {
        attn_bwd_dq_kernel<false><<<dim3(np, n_q_heads, U), NTHREADS, SMEM, st>>>(tm[0], tm[1], tm[2], tm[3], pp);
        BR_CHECK_LAUNCH();
    }
    // suffix dQ (+ suffix delta)
    BwdParams ps = p;
    ps.B = R; ps.L = Lp + Ls; ps.kv_end = kv_end;
    attn_bwd_dq_kernel<true><<<dim3(ns, n_q_heads, R), NTHREADS, SMEM, st>>>(tm[0], tm[1], tm[2], tm[3], ps);
    BR_CHECK_LAUNCH();
    // suffix dK / dV: dense kernel on [R, Ls], windows in suffix coordinates
    shift_windows_kernel<<<(R + 127) / 128, 128, 0, st>>>(kv_start, kv_end, G, R, Lp, ks_s, ke_s);
    BR_CHECK_LAUNCH();
    BwdParams pk = p;
    pk.B = R; pk.L = Ls; pk.lse = lse_suffix; pk.delta = delta_s; pk.kv_start = ks_s; pk.kv_end = ke_s;
    pk.o = p.o + sfx0 * ldo; pk.dout = p.dout + sfx0 * lddo;
    pk.dq = p.dq + sfx0 * lddq; pk.dk = p.dk + sfx0 * lddk; pk.dv = p.dv + sfx0 * lddv;
    attn_bwd_dkv_kernel<false><<<dim3(ns, n_kv_heads, R), NTHREADS, SMEM, st>>>(tm_s[0], tm_s[1], tm_s[2], tm_s[3], pk);
    BR_CHECK_LAUNCH();
    // prefix dK / dV: prefix queries, then the G suffixes of the group
    if (np > 0) {
        attn_bwd_dkv_kernel<true><<<dim3(np, n_kv_heads, U), NTHREADS, SMEM, st>>>(tm[0], tm[1], tm[2], tm[3], pp);
        BR_CHECK_LAUNCH();
    }
    return BR_OK;
}
