// Flash attention forward on wgmma / TMA (sm_90a): causal GQA decoder rows (D=128) and bidirectional encoder rows (D=64).
// Replaces the SDPA call HF reaches from Qwen3Attention.forward (qwen3/modeling_qwen3.py:255-263) and EsmSelfAttention.forward
// (esm/modeling_esm.py:349-359); SURVEY.md §2.3 K1/K5.  Dense [B, L] token-major rows, row b attends keys j in
// [kv_start[b], kv_end[b]) (one contiguous window: left pads / post-EOS tail are outside), j <= i when causal; optional
// log-sum-exp output for the backward.
//
// Shared-prefix mode (SHARED = true, causal D = 128 only; br_attn_fwd_shared): the token buffer holds U groups of G rows as
// [U * Lp prefix rows | R = U * G suffixes of Ls rows], Lp a multiple of 64.  A CTA handles a query tile of suffix row r; key tiles
// j < Lp / 64 come from group r / G's prefix rows, later ones from row r's suffix.  Tiles, tile order and masks are those of the dense
// kernel on the equivalent [R, Lp + Ls] row, so O and the log-sum-exp are bit-identical to it.
//
// One CTA = one warpgroup = one 64-query tile of one (batch row, query head); 80 KB of shared memory at D = 128 (two CTAs per SM),
// 48 KB at D = 64 (four).  Thread 0 issues the TMA
// loads: the Q tile once, K and V tiles (64 keys x D, 128B-swizzled 64-column boxes) through a two-stage ring, so tile t+1 lands
// while tile t is computed.  Per key tile:
//   S = Q K^T      wgmma m64n64k16, both operands K-major in shared memory, scores in registers
//   softmax        online, in registers: a quad of lanes shares a query row (shuffle reductions), exp2 in the log2 domain
//   O += P V       wgmma m64nDk16 with P as the REGISTER A operand (the score fragment re-packed to bf16, no shared-memory
//                  round trip) and V as an MN-major shared-memory operand (the TMA tile [keys, d] as it lands: no transposed copy)
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "wgmma.cuh"

namespace {

constexpr int BM = 64, BN = 64, NTHREADS = 128;

struct FwdParams {
    bf16* o; long long ldo;
    float* lse;                  // [B, Hq, L] or null
    int B, L, Hq, Hkv;
    const int *kv_start, *kv_end;
    float scale_log2;            // softmax scale * log2(e)
    // shared-prefix mode: L = Lp + Ls, B = R suffix rows, kv_start per group ([R / G]), kv_end per row, lse [R, Hq, Ls]
    int G, Lp, Ls;
    long long sfx0;              // first suffix row of the buffer (U * Lp)
};

__device__ __forceinline__ float ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

template <int D>
struct SL {
    static constexpr int NB = D / 64;                  // 64-column (128-byte) swizzled blocks per row
    static constexpr int BLK = 64 * 128;               // bytes of one [64 rows x 64 cols] block
    static constexpr int TILE = NB * BLK;              // a [64 x D] bf16 tile
    static constexpr int OFF_Q = 0;
    static constexpr int OFF_K = TILE;                 // 2 stages
    static constexpr int OFF_V = OFF_K + 2 * TILE;     // 2 stages
    static constexpr int OFF_BAR = OFF_V + 2 * TILE;
    static constexpr int TOTAL = OFF_BAR + 64 + 1024;
};

template <int D, bool CAUSAL, bool SHARED>
__global__ void __launch_bounds__(NTHREADS, 2)
attn_fwd_tc5_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const FwdParams p) {
    using L = SL<D>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
    uint64_t* kv_full = q_full + 1;                // 2

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int qb = (SHARED ? p.Lp / BM : 0) + gridDim.x - 1 - blockIdx.x;     // heavy (late) causal tiles first
    const int h = blockIdx.y, b = blockIdx.z;
    const int hk = h / (p.Hq / p.Hkv);
    const int q0 = qb * BM;
    const int ks = p.kv_start ? p.kv_start[SHARED ? b / p.G : b] : 0;
    const int ke = p.kv_end ? p.kv_end[b] : p.L;
    int last_key = ke - 1;
    if (CAUSAL) last_key = min(last_key, q0 + BM - 1);
    const int jb_lo = ks / BN;
    int jb_hi = last_key >= 0 ? last_key / BN : -1;          // inclusive
    if (ke <= ks) jb_hi = jb_lo - 1;
    const int n_tiles = max(0, jb_hi - jb_lo + 1);

    // buffer row of position i of this CTA's row (queries and outputs: i >= Lp in shared mode)
    auto tok_row = [&](int i) -> long long { return SHARED ? p.sfx0 + (long long)b * p.Ls + (i - p.Lp) : (long long)b * p.L + i; };
    auto load_kv = [&](int t) {
        const int st = t & 1, j0 = (jb_lo + t) * BN;
        const int row_k = SHARED ? (j0 < p.Lp ? (b / p.G) * p.Lp + j0 : (int)tok_row(j0)) : b * p.L + j0;
        br::mbar_expect_tx(&kv_full[st], 2 * L::TILE);
#pragma unroll
        for (int nb = 0; nb < L::NB; ++nb) {
            br::tma_load_2d(smem + L::OFF_K + st * L::TILE + nb * L::BLK, &tmK, &kv_full[st], hk * D + nb * 64, row_k);
            br::tma_load_2d(smem + L::OFF_V + st * L::TILE + nb * L::BLK, &tmV, &kv_full[st], hk * D + nb * 64, row_k);
        }
    };
    if (tid == 0) {
        br::tma_prefetch_desc(&tmQ); br::tma_prefetch_desc(&tmK); br::tma_prefetch_desc(&tmV);
        br::mbar_init(q_full, 1); br::mbar_init(&kv_full[0], 1); br::mbar_init(&kv_full[1], 1);
        br::mbar_fence_init();
        if (n_tiles > 0) {
            br::mbar_expect_tx(q_full, L::TILE);
#pragma unroll
            for (int nb = 0; nb < L::NB; ++nb) br::tma_load_2d(smem + L::OFF_Q + nb * L::BLK, &tmQ, q_full, h * D + nb * 64, (int)tok_row(q0));
            load_kv(0);
            if (n_tiles > 1) load_kv(1);
        }
    }
    __syncthreads();

    // fragment rows of this thread: r0 and r0 + 8 of the tile; columns 8i + cq + {0, 1}
    const int r0 = warp * 16 + (lane >> 2), cq = 2 * (lane & 3);
    float o_acc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o_acc[i] = 0.f;
    float m_used[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};      // running maximum in units of RAW scores * scale_log2
    const uint32_t q_addr = br::smem_u32(smem + L::OFF_Q);
    if (n_tiles > 0) br::mbar_wait(q_full, 0);
    for (int t = 0; t < n_tiles; ++t) {
        const int st = t & 1;
        const int nbase = (jb_lo + t) * BN;
        const uint32_t k_addr = br::smem_u32(smem + L::OFF_K + st * L::TILE), v_addr = br::smem_u32(smem + L::OFF_V + st * L::TILE);
        br::mbar_wait(&kv_full[st], (t >> 1) & 1);
        float s[BN / 2];
        br::wg_fence();
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
            const uint32_t off = (kk >> 2) * L::BLK + (kk & 3) * 32;
            br::wgmma_ss<BN>(s, br::wg_desc_k(q_addr + off), br::wg_desc_k(k_addr + off), kk != 0);
        }
        br::wg_commit();
        br::wg_wait<0>();
        br::wg_fence_operand(s);
        const bool need_mask = (nbase < ks) || (nbase + BN > ke) || (CAUSAL && nbase + BN - 1 > q0);
        if (need_mask) {
#pragma unroll
            for (int i = 0; i < BN / 8; ++i)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int j = nbase + 8 * i + cq + e, ig = q0 + r0 + 8 * hh;
                        if (!((j >= ks) && (j < ke) && (!CAUSAL || j <= ig))) s[4 * i + 2 * hh + e] = -INFINITY;
                    }
        }
        float alpha[2], ms[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * hh], s[4 * i + 2 * hh + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_used[hh], mx * p.scale_log2);     // scale > 0: the max commutes with the scaling
            alpha[hh] = 1.f;
            if (m_new > m_used[hh]) { alpha[hh] = (m_used[hh] == -INFINITY) ? 0.f : ex2(m_used[hh] - m_new); m_used[hh] = m_new; }
            ms[hh] = (m_used[hh] == -INFINITY) ? 0.f : m_used[hh];
        }
        float rs[2] = {0.f, 0.f};
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pr = ex2(fmaf(s[4 * i + 2 * hh + e], p.scale_log2, -ms[hh]));
                    s[4 * i + 2 * hh + e] = pr;
                    rs[hh] += pr;
                }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) l[hh] = l[hh] * alpha[hh] + rs[hh];
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) { o_acc[4 * i + 2 * hh] *= alpha[hh]; o_acc[4 * i + 2 * hh + 1] *= alpha[hh]; }
        br::wg_fence();
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk) {
            const uint32_t a[4] = {br::pack_bf16(s[8 * kk + 0], s[8 * kk + 1]), br::pack_bf16(s[8 * kk + 2], s[8 * kk + 3]),
                                   br::pack_bf16(s[8 * kk + 4], s[8 * kk + 5]), br::pack_bf16(s[8 * kk + 6], s[8 * kk + 7])};
            // 16 keys = 2 groups of 8 rows (SBO = 1024 B); the D/64 blocks of 64 d-columns are L::BLK bytes apart (LBO)
            br::wgmma_rs<D, 1>(o_acc, a, br::wg_desc_mn(v_addr + kk * 2048, L::BLK, 1024), 1);
        }
        br::wg_commit();
        br::wg_wait<0>();
        br::wg_fence_operand(o_acc);
        __syncthreads();                                        // every thread's products of stage st have retired
        if (tid == 0 && t + 2 < n_tiles) load_kv(t + 2);
    }
    // ---- epilogue: O / l -> bf16 rows, log-sum-exp
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        float lt = l[hh];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        const int i_glob = q0 + r0 + 8 * hh;
        if (i_glob >= p.L) continue;
        const float inv = lt > 0.f ? 1.f / lt : 0.f;
        bf16* orow = p.o + tok_row(i_glob) * p.ldo + (long long)h * D;
#pragma unroll
        for (int i = 0; i < D / 8; ++i)
            *reinterpret_cast<uint32_t*>(orow + 8 * i + cq) = br::pack_bf16(o_acc[4 * i + 2 * hh] * inv, o_acc[4 * i + 2 * hh + 1] * inv);
        if (p.lse && (lane & 3) == 0) {
            const float LN2 = 0.6931471805599453f;
            const long long li = SHARED ? ((long long)b * p.Hq + h) * p.Ls + i_glob - p.Lp : ((long long)b * p.Hq + h) * p.L + i_glob;
            p.lse[li] = lt > 0.f ? m_used[hh] * LN2 + logf(lt) : INFINITY;
        }
    }
}

template <int D, bool CAUSAL, bool SHARED = false>
int launch(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const FwdParams& p, cudaStream_t st) {
    using L = SL<D>;
    auto kern = attn_fwd_tc5_kernel<D, CAUSAL, SHARED>;
    static bool done = false;
    if (!done) {
        BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
        BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));       // several CTAs per SM
        done = true;
    }
    dim3 grid(((SHARED ? p.Ls : p.L) + BM - 1) / BM, p.Hq, p.B);
    kern<<<grid, NTHREADS, L::TOTAL, st>>>(tq, tk, tv, p);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

}  // namespace

int br_attn_fwd_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo, float* lse,
                         int B, int L, int n_q_heads, int n_kv_heads, int head_dim, const int32_t* kv_start, const int32_t* kv_end,
                         float scale, int causal, cudaStream_t st) {
    FwdParams p = {};
    p.o = (bf16*)o; p.ldo = ldo; p.lse = lse; p.B = B; p.L = L; p.Hq = n_q_heads; p.Hkv = n_kv_heads;
    p.kv_start = kv_start; p.kv_end = kv_end; p.scale_log2 = scale * 1.4426950408889634f;
    BR_CHECK_ARG(((uintptr_t)q % 16 == 0) && ((uintptr_t)k % 16 == 0) && ((uintptr_t)v % 16 == 0) && ((uintptr_t)o % 16 == 0),
                 "attn_fwd: q/k/v/o must be 16-byte aligned");
    CUtensorMap tq, tk, tv;
    int rc;
    const uint64_t rows = (uint64_t)B * L;
    if ((rc = br_make_tmap_2d_bf16(&tq, q, rows, (uint64_t)n_q_heads * head_dim, ldq, BM))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tk, k, rows, (uint64_t)n_kv_heads * head_dim, ldk, BN))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tv, v, rows, (uint64_t)n_kv_heads * head_dim, ldv, BN))) return rc;
    if (head_dim == 128) return causal ? launch<128, true>(tq, tk, tv, p, st) : launch<128, false>(tq, tk, tv, p, st);
    return causal ? launch<64, true>(tq, tk, tv, p, st) : launch<64, false>(tq, tk, tv, p, st);
}

int br_attn_fwd_shared_tc5_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                                float* lse_prefix, float* lse_suffix, int U, int G, int Lp, int Ls, int n_q_heads, int n_kv_heads,
                                const int32_t* kv_start, const int32_t* kv_end, float scale, cudaStream_t st) {
    BR_CHECK_ARG(((uintptr_t)q % 16 == 0) && ((uintptr_t)k % 16 == 0) && ((uintptr_t)v % 16 == 0) && ((uintptr_t)o % 16 == 0),
                 "attn_fwd_shared: q/k/v/o must be 16-byte aligned");
    const uint64_t rows = (uint64_t)U * Lp + (uint64_t)U * G * Ls;
    CUtensorMap tq, tk, tv;
    int rc;
    if ((rc = br_make_tmap_2d_bf16(&tq, q, rows, (uint64_t)n_q_heads * 128, ldq, BM))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tk, k, rows, (uint64_t)n_kv_heads * 128, ldk, BN))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tv, v, rows, (uint64_t)n_kv_heads * 128, ldv, BN))) return rc;
    FwdParams p = {};
    p.o = (bf16*)o; p.ldo = ldo; p.Hq = n_q_heads; p.Hkv = n_kv_heads; p.kv_start = kv_start; p.scale_log2 = scale * 1.4426950408889634f;
    if (Lp > 0) {                                   // prefix rows: the dense kernel on [U, Lp] (prefix queries see prefix keys only)
        p.lse = lse_prefix; p.B = U; p.L = Lp; p.kv_end = nullptr;
        if ((rc = launch<128, true>(tq, tk, tv, p, st))) return rc;
    }
    p.lse = lse_suffix; p.B = U * G; p.L = Lp + Ls; p.kv_end = kv_end;
    p.G = G; p.Lp = Lp; p.Ls = Ls; p.sfx0 = (long long)U * Lp;
    return launch<128, true, true>(tq, tk, tv, p, st);
}
