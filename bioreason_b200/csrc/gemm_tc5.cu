// wgmma / TMA GEMM for sm_90a:  D[M,N] = alpha * (A[M,K] . B[N,K]^T  (+ A2[M,K2] . B2[N,K2]^T)) (+bias)(+residual)
//
// Replaces every nn.Linear / lm_head matmul the reference reaches through HF (SURVEY.md §2.3 K1,K2,K5,K6,K12):
// both operands are K-major (nn.Linear weight layout [out, in]), bf16 in, fp32 accumulate in registers.
//
// Structure (one persistent CTA per SM, 288 threads, a 128 x BN tile with BN = 128 or 256 chosen per problem in run_gemm):
//   warp 8      TMA producer   : cp.async.bulk.tensor 2-D, 128B-swizzled 128x64 (A) and BNx64 (B) tiles, NSTAGE ring
//   warps 0..7  two consumer warpgroups: each issues wgmma.mma_async m64nBNk16 for its 64 rows of the 128 x BN tile (one
//                                wgmma group kept in flight; a stage goes back to the producer as soon as its products retire),
//                                then runs the fused epilogue straight from the register fragment
// Every output element accumulates over K in the same k16 order at either width, and the epilogues round at the same points, so
// the two tile widths give bit-identical results.
// LoRA dropout (MASK): the second K segment u . A of the dX GEMM is formed one projection (r-wide K block) at a time in a temporary
// accumulator, multiplied by that projection's counter-based mask and 1 / (1 - p_eff) in registers, and added to the main accumulator
// before the usual epilogue (one rounding, no extra HBM traffic).
// Epilogue modes: plain (+bias, +residual, gated-SiLU on interleaved column pairs, fp32/bf16 out, row scatter),
// online log-sum-exp partials + target-logit gather (lm_head; logits never reach HBM; optionally with entropy partials),
// and softmax-gradient tiles.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "lora_dropout.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int NTHREADS = 288;

enum { MODE_STD = 0, MODE_LSE = 1, MODE_DLOGITS = 2, MODE_LSE_ENT = 3 };   // MODE_LSE_ENT: MODE_LSE + the entropy partials

struct GemmParams {
    int M, N, K, K2;
    int ldd;                 // elements
    void* D;
    const void* bias; int bias_f32;
    const bf16* residual; long long ldr;
    float alpha;
    int act;                 // 1: gated SiLU over column blocks of 16 = 8 gate | 8 up -> 8 outputs
    int out_f32;
    const int* row_map;
    bf16* aux; long long ld_aux;   // act==1: raw (pre-activation) accumulator pairs, bf16 [M, N]
    // MODE_LSE / MODE_DLOGITS
    const int* target;       // [M] class index per row (or <0)
    float* pmax; float* psum; float* tgt_logit;   // [M, n_tiles_n], [M, n_tiles_n], [M]
    const float* lse; const float* gscale;        // [M]
    int n_tiles_m, n_tiles_n;      // 128-row and 128-column tiles; a BN-wide tile spans BN / 128 column tiles
                                   // (MODE_LSE writes one partial per 128-column tile: [M, n_tiles_n])
    int group_m;             // m-blocks per raster group (see tile_coords)
    br::DropParams drop;     // MASK: dropout of the second segment's projections
    float* pent;             // MODE_LSE_ENT: [M, n_tiles_n] u_t = sum over the tile of exp(z - m_t) (z - m_t)  (<= 0)
};

template <int BN>
struct SmemLayout {
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int NSTAGE = BN == 128 ? 6 : 4;        // 6 x 32 KB or 4 x 48 KB of the 227 KB a block may use
    static constexpr int TILE_BYTES = NSTAGE * STAGE_BYTES;
    static constexpr int TOTAL = TILE_BYTES + 256 + 1024;   // + barriers + alignment slack
};

__device__ __forceinline__ void tile_coords(int tile, int ntm, int ntn, int GROUP_M, int& mb, int& nb) {
    // grouped rasterisation: GROUP_M m-blocks x all n-blocks per group.  The group's A panel (GROUP_M x 128 x K, sized by the host to
    // about a third of L2) stays L2-resident while every B panel streams past it once, so B is re-read from DRAM once per GROUP.
    int per_group = GROUP_M * ntn;
    int g = tile / per_group;
    int first_m = g * GROUP_M;
    int gsize = min(GROUP_M, ntm - first_m);
    int r = tile - g * per_group;
    mb = first_m + (r % gsize);
    nb = r / gsize;
}

__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16(x)); }

// One BK block of the LoRA segment under dropout: for each projection whose r-wide K slice lies in the block, tmp = u_j . A_j (its k16
// steps), then acc += m_j * inv_keep * tmp over the thread's fragment.  Retires every outstanding wgmma of the tile first.
template <int BN>
__device__ __forceinline__ void masked_segment(float (&acc)[BN / 2], uint64_t adesc, uint64_t bdesc, int k0, int mb, int nb, int wg,
                                               const GemmParams& p) {
    const int lane = threadIdx.x & 31, q = lane & 3;
    const long long grow = p.drop.row0 + mb * BM + wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
    const int cg0 = (nb * BN) >> 3;
    br::wg_wait<0>();
    br::wg_fence_operand(acc);
    for (int kk = 0; kk < BK / 16;) {
        const int kc = k0 + 16 * kk;
        if (kc >= p.K2) break;
        const int jb = kc / p.drop.r;
        const int nk = min(p.drop.r - (kc - jb * p.drop.r), BK - 16 * kk) >> 4;     // k16 steps of projection jb in this block
        float tmp[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) tmp[i] = 0.f;
        br::wg_fence();
        for (int t = 0; t < nk; ++t) br::wgmma_ss<BN>(tmp, adesc + 2 * (kk + t), bdesc + 2 * (kk + t), 1);
        br::wg_commit();
        br::wg_wait<0>();
        br::wg_fence_operand(tmp);
        const int j = p.drop.proj + jb;
#pragma unroll
        for (int set = 0; set < BN / 16; ++set) {                   // 2 rows x BN / 8 column groups = BN / 4 groups, 4 per set
            // groups g = 0..3 of this set: column group 2 set + (g >> 1), row + 8 (g & 1); lane q draws group q
            uint32_t w[4];
            br::quad_words(br::drop_group(p.drop, grow + 8 * (q & 1), cg0 + 2 * set + (q >> 1), j), w);
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const int e = 4 * (2 * set + (g >> 1)) + 2 * (g & 1);
                acc[e] += br::keep_lo(w[g], p.drop.T) ? tmp[e] * p.drop.inv_keep : 0.f;
                acc[e + 1] += br::keep_hi(w[g], p.drop.T) ? tmp[e + 1] * p.drop.inv_keep : 0.f;
            }
        }
        kk += nk;
    }
}

template <int BN, int MODE, bool MASK>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc5_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                const GemmParams p) {
    static_assert(BN == 128 || BN == 256, "tile width");
    static_assert(!MASK || BN == 128, "the masked LoRA segment runs on 128-wide tiles");
    constexpr int NSUB = BN / 128;                          // 128-column tiles per tile
    using L = SmemLayout<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::TILE_BYTES);
    uint64_t* empty_bar = full_bar + L::NSTAGE;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.n_tiles_m * ((p.n_tiles_n + NSUB - 1) / NSUB);
    const int kb1 = (p.K + BK - 1) / BK;
    const int kb2 = (p.K2 + BK - 1) / BK;
    const int num_kb = kb1 + kb2;

    if (threadIdx.x == 0) {
        br::tma_prefetch_desc(&tmA);
        br::tma_prefetch_desc(&tmB);
        if (kb2) { br::tma_prefetch_desc(&tmA2); br::tma_prefetch_desc(&tmB2); }
        for (int s = 0; s < L::NSTAGE; ++s) { br::mbar_init(&full_bar[s], 1); br::mbar_init(&empty_bar[s], 2); }
        br::mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                int mb, nb; tile_coords(tile, p.n_tiles_m, (p.n_tiles_n + NSUB - 1) / NSUB, p.group_m, mb, nb);
                for (int kb = 0; kb < num_kb; ++kb) {
                    br::mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* sa = smem + s * L::STAGE_BYTES;
                    uint8_t* sb = sa + L::A_BYTES;
                    br::mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
                    if (kb < kb1) {
                        br::tma_load_2d(sa, &tmA, &full_bar[s], kb * BK, mb * BM);
                        br::tma_load_2d(sb, &tmB, &full_bar[s], kb * BK, nb * BN);
                    } else {
                        br::tma_load_2d(sa, &tmA2, &full_bar[s], (kb - kb1) * BK, mb * BM);
                        br::tma_load_2d(sb, &tmB2, &full_bar[s], (kb - kb1) * BK, nb * BN);
                    }
                    if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
                }
            }
        }
        return;
    }
    // ===================== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the 128 x BN tile =====================
    const int wg = warp >> 2;
    const int wt = threadIdx.x & 127;
    int s = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int mb, nb; tile_coords(tile, p.n_tiles_m, (p.n_tiles_n + NSUB - 1) / NSUB, p.group_m, mb, nb);
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
            br::mbar_wait(&full_bar[s], ph);
            const uint32_t sa = br::smem_u32(smem + s * L::STAGE_BYTES);
            const uint64_t adesc = br::wg_desc_k(sa + wg * 64 * 128);
            const uint64_t bdesc = br::wg_desc_k(sa + L::A_BYTES);
            if constexpr (MASK) {
                if (kb >= kb1) {
                    masked_segment<BN>(acc, adesc, bdesc, (kb - kb1) * BK, mb, nb, wg, p);
                    if (wt == 0) br::mbar_arrive(&empty_bar[prev]);       // masked_segment retired every product: release the previous stage
                    prev = s;
                    if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
                    continue;
                }
            }
            br::wg_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) br::wgmma_ss<BN>(acc, adesc + 2 * k, bdesc + 2 * k, 1);
            br::wg_commit();
            if (kb > 0) {                                  // the previous stage's products have retired: hand it back
                br::wg_wait<1>();
                if (wt == 0) br::mbar_arrive(&empty_bar[prev]);
            }
            prev = s;
            if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
        }
        br::wg_wait<0>();
        br::wg_fence_operand(acc);
        if (wt == 0) br::mbar_arrive(&empty_bar[prev]);

        // ---- epilogue straight from the accumulator fragment: thread holds rows r0, r0 + 8 and column pairs 8i + 2 (lane % 4)
        const int r0 = mb * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int n0 = nb * BN;
        const int cq = 2 * (lane & 3);
        if constexpr (MODE == MODE_STD) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int row = r0 + 8 * hh;
                if (row >= p.M) continue;
                const long long orow = p.row_map ? (long long)p.row_map[row] : (long long)row;
                if (orow < 0) continue;
                float v[BN / 4];
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    v[2 * i] = acc[4 * i + 2 * hh] * p.alpha;
                    v[2 * i + 1] = acc[4 * i + 2 * hh + 1] * p.alpha;
                    const int col = n0 + 8 * i + cq;
                    if (p.bias && n0 + 8 * i < p.N) {
                        if (p.bias_f32) {
                            const float* b = reinterpret_cast<const float*>(p.bias) + col;
                            v[2 * i] += __ldg(b); v[2 * i + 1] += __ldg(b + 1);
                        } else {
                            const bf16* b = reinterpret_cast<const bf16*>(p.bias) + col;
                            v[2 * i] += __bfloat162float(b[0]); v[2 * i + 1] += __bfloat162float(b[1]);
                        }
                    }
                }
                if (p.act == 1) {
#pragma unroll
                    for (int j = 0; j < BN / 16; ++j) {
                        if (n0 + 16 * j >= p.N) break;
                        if (p.aux) {
                            bf16* a = p.aux + orow * p.ld_aux + n0 + 16 * j + cq;
                            *reinterpret_cast<uint32_t*>(a) = br::pack_bf16(v[4 * j], v[4 * j + 1]);
                            *reinterpret_cast<uint32_t*>(a + 8) = br::pack_bf16(v[4 * j + 2], v[4 * j + 3]);
                        }
                        // columns come in blocks of 16 = 8 gate | 8 up (packing.py); HF computes act_fn(gate) in bf16 then multiplies:
                        // round at the same places
                        float o[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const float g = rbf(v[4 * j + e]), u = rbf(v[4 * j + 2 + e]);
                            o[e] = rbf(g / (1.f + __expf(-g))) * u;
                        }
                        bf16* d = reinterpret_cast<bf16*>(p.D) + orow * (long long)p.ldd + (n0 >> 1) + 8 * j + cq;
                        *reinterpret_cast<uint32_t*>(d) = br::pack_bf16(o[0], o[1]);
                    }
                    continue;
                }
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    if (n0 + 8 * i >= p.N) break;
                    const int col = n0 + 8 * i + cq;
                    float x0 = v[2 * i], x1 = v[2 * i + 1];
                    if (p.residual) {
                        // nn.Linear output is rounded to bf16 before the residual add in HF
                        const float2 r = br::unpack_bf16(__ldg(reinterpret_cast<const unsigned int*>(p.residual + orow * p.ldr + col)));
                        x0 = rbf(x0) + r.x; x1 = rbf(x1) + r.y;
                    }
                    if (p.out_f32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.D) + orow * (long long)p.ldd + col) = make_float2(x0, x1);
                    else *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.D) + orow * (long long)p.ldd + col) = br::pack_bf16(x0, x1);
                }
            }
        } else if constexpr (MODE == MODE_LSE || MODE == MODE_LSE_ENT) {
            // per-row max / sum-exp over each 128-column tile (the four lanes of a quad share a row) + target-logit pick.  A 256-wide
            // tile writes its two halves as two partials, so the partials and their combine do not depend on the tile width.
            // MODE_LSE_ENT also sums exp(z - m) (z - m) from the same exps; every term is <= 0, so the partial keeps its sign.
#pragma unroll
            for (int h = 0; h < NSUB; ++h) {
                const int nh = n0 + 128 * h;
                if (NSUB > 1 && nh >= p.N) break;           // the last 256-wide tile may cover a single 128-column tile
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int row = r0 + 8 * hh;
                    const bool row_ok = row < p.M;
                    const int tgt = row_ok ? p.target[row] : -1;
                    float mx = -INFINITY;
#pragma unroll
                    for (int i = 0; i < 16; ++i)
                        if (nh + 8 * i < p.N) mx = fmaxf(mx, fmaxf(acc[64 * h + 4 * i + 2 * hh], acc[64 * h + 4 * i + 2 * hh + 1]) * p.alpha);
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    float sm = 0.f, un = 0.f;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        if (nh + 8 * i >= p.N) continue;
                        const int col = nh + 8 * i + cq;
                        const float x0 = acc[64 * h + 4 * i + 2 * hh] * p.alpha, x1 = acc[64 * h + 4 * i + 2 * hh + 1] * p.alpha;
                        if constexpr (MODE == MODE_LSE_ENT) {
                            const float d0 = x0 - mx, d1 = x1 - mx;
                            const float e0 = __expf(d0), e1 = __expf(d1);
                            sm += e0 + e1;
                            un += e0 * d0 + e1 * d1;
                        } else {
                            sm += __expf(x0 - mx) + __expf(x1 - mx);
                        }
                        if (col == tgt) p.tgt_logit[row] = x0;
                        if (col + 1 == tgt) p.tgt_logit[row] = x1;
                    }
                    sm += __shfl_xor_sync(0xffffffffu, sm, 1);
                    sm += __shfl_xor_sync(0xffffffffu, sm, 2);
                    if constexpr (MODE == MODE_LSE_ENT) {
                        un += __shfl_xor_sync(0xffffffffu, un, 1);
                        un += __shfl_xor_sync(0xffffffffu, un, 2);
                    }
                    if (row_ok && (lane & 3) == 0) {
                        p.pmax[(long long)row * p.n_tiles_n + nb * NSUB + h] = mx;
                        p.psum[(long long)row * p.n_tiles_n + nb * NSUB + h] = sm;
                        if constexpr (MODE == MODE_LSE_ENT) p.pent[(long long)row * p.n_tiles_n + nb * NSUB + h] = un;
                    }
                }
            }
        } else {
            // dlogits[m, n] = gscale[m] * (onehot(target[m])[n] - exp(logit - lse[m]))   (bf16 out)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int row = r0 + 8 * hh;
                if (row >= p.M) continue;
                const int tgt = p.target[row];
                const float lse = p.lse[row], gs = p.gscale[row];
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    if (n0 + 8 * i >= p.N) break;
                    const int col = n0 + 8 * i + cq;
                    const float d0 = gs * ((col == tgt ? 1.f : 0.f) - __expf(acc[4 * i + 2 * hh] * p.alpha - lse));
                    const float d1 = gs * ((col + 1 == tgt ? 1.f : 0.f) - __expf(acc[4 * i + 2 * hh + 1] * p.alpha - lse));
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.D) + (long long)row * p.ldd + col) = br::pack_bf16(d0, d1);
                }
            }
        }
    }
}

// lse[m] = log sum_t psum[m,t] * exp(pmax[m,t] - gmax) + gmax ; logp[m] = tgt_logit[m] - lse[m]
__global__ void lse_combine_kernel(const float* __restrict__ pmax, const float* __restrict__ psum, const float* __restrict__ tgt_logit,
                                   const int* __restrict__ target, int M, int nt, float* __restrict__ lse, float* __restrict__ logp) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    int lane = threadIdx.x & 31;
    float mx = -INFINITY;
    for (int t = lane; t < nt; t += 32) mx = fmaxf(mx, pmax[(long long)row * nt + t]);
    mx = br::warp_max(mx);
    float s = 0.f;
    for (int t = lane; t < nt; t += 32) s += psum[(long long)row * nt + t] * __expf(pmax[(long long)row * nt + t] - mx);
    s = br::warp_sum(s);
    if (lane == 0) {
        float l = logf(s) + mx;
        if (lse) lse[row] = l;
        if (logp) logp[row] = (target[row] >= 0) ? tgt_logit[row] - l : 0.f;
    }
}

// lse_combine_kernel plus the entropy H = -sum_j p_j log p_j of the row (p = softmax of the row's logits).  With M = max_t m_t and
// r_t = exp(m_t - M):  S = sum_t s_t r_t,  U = sum_t r_t (u_t + (m_t - M) s_t),  H = log S - U / S.  S and lse are formed exactly as
// lse_combine_kernel forms them (same loops, same order), so lse and logp are bit-identical to it.  Every term of U is <= 0 and
// S >= 1 (the maximal tile contributes s_t >= exp(0) = 1), so both terms of H are >= 0 and H >= 0 in floating point as well.
__global__ void lse_entropy_combine_kernel(const float* __restrict__ pmax, const float* __restrict__ psum, const float* __restrict__ pent,
                                           const float* __restrict__ tgt_logit, const int* __restrict__ target, int M, int nt,
                                           float* __restrict__ lse, float* __restrict__ logp, float* __restrict__ ent) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    int lane = threadIdx.x & 31;
    float mx = -INFINITY;
    for (int t = lane; t < nt; t += 32) mx = fmaxf(mx, pmax[(long long)row * nt + t]);
    mx = br::warp_max(mx);
    float s = 0.f, u = 0.f;
    for (int t = lane; t < nt; t += 32) {
        const float dm = pmax[(long long)row * nt + t] - mx;
        const float r = __expf(dm), st = psum[(long long)row * nt + t];
        s += st * r;
        u += r * (pent[(long long)row * nt + t] + dm * st);
    }
    s = br::warp_sum(s);
    u = br::warp_sum(u);
    if (lane == 0) {
        const float ls = logf(s);
        float l = ls + mx;
        if (lse) lse[row] = l;
        if (logp) logp[row] = (target[row] >= 0) ? tgt_logit[row] - l : 0.f;
        ent[row] = ls - u / s;
    }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(f);
    }
    return fn;
}

template <int BN, int MODE, bool MASK = false>
int launch(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& a2, const CUtensorMap& b2, const GemmParams& p, cudaStream_t st) {
    auto kern = gemm_tc5_kernel<BN, MODE, MASK>;
    static bool attr_set = false;
    if (!attr_set) {
        BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout<BN>::TOTAL));
        attr_set = true;
    }
    int tiles = p.n_tiles_m * ((p.n_tiles_n + BN / 128 - 1) / (BN / 128));
    int grid = tiles < br_num_sms() ? tiles : br_num_sms();
    kern<<<grid, NTHREADS, SmemLayout<BN>::TOTAL, st>>>(a, b, a2, b2, p);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

template <int BN>
int launch_mode(int mode, const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& a2, const CUtensorMap& b2, const GemmParams& p,
                cudaStream_t st) {
    if (mode == MODE_STD) return launch<BN, MODE_STD>(a, b, a2, b2, p, st);
    if (mode == MODE_LSE) return launch<BN, MODE_LSE>(a, b, a2, b2, p, st);
    if (mode == MODE_LSE_ENT) return launch<BN, MODE_LSE_ENT>(a, b, a2, b2, p, st);
    return launch<BN, MODE_DLOGITS>(a, b, a2, b2, p, st);
}

int run_gemm(int mode, const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, const void* A2, int64_t lda2,
             const void* B2, int64_t ldb2, int K2, GemmParams& p, cudaStream_t st, bool masked = false) {
    BR_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
    BR_CHECK_ARG(N % 8 == 0 && K % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0, "gemm: N, K, lda, ldb must be multiples of 8");
    BR_CHECK_ARG(((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0), "gemm: operands must be 16-byte aligned");
    p.M = M; p.N = N; p.K = K; p.K2 = (A2 && B2) ? K2 : 0;
    p.n_tiles_m = (M + BM - 1) / BM;
    p.n_tiles_n = (N + 127) / 128;
    // Tile width.  Per k16, each warpgroup reads its A slice and the whole B slice from shared memory; m64n256 does twice the math
    // of m64n128 for the same A read, and a 256-wide CTA loads each A tile from L2 once per 256 output columns instead of once per
    // 128 (1.1-1.3x the TFLOP/s on the training shapes, DESIGN.md section 5).  The 128 x 256 tile has half as many tiles to spread over the SMs and a 4-stage ring, so it is used only where the
    // tiles still fill two waves of the persistent grid and the main loop dominates the tile: N >= 256, K >= 512 and at least
    // 2 x SMs 256-wide tiles.  That takes the training-pass linears at the trainer's chunk sizes (4 x 2364 dense rows, 6368
    // shared-prefix rows) and the lm_head.  The LoRA down / up products (N = r x projections <= 96), the merged-weight rebuild
    // (K = r), the DNA encoder, the projector and one-prompt prefills of the 2560-wide outputs keep 128 x 128.  The masked LoRA
    // segment (dropout) always runs 128-wide: it needs a second accumulator of the tile's width.
    const bool wide = !masked && N >= 256 && K >= 512 && (long long)p.n_tiles_m * ((N + 255) / 256) >= 2ll * br_num_sms();
    const int bn = wide ? 256 : 128;
    {   // A panel of one raster group ~ 16 MB of the 50 MB L2 (the concurrently streaming B panels and the outputs need the rest).
        // The rule counts 128-row A blocks, so it is the same at both tile widths: B is re-read from DRAM once per group at either
        // width, and the B panels of one wave of 256-wide tiles, (SMs / group_m) x 256 x K x 2 bytes, stay within the rest of L2 up
        // to K = 4096 (beyond that, at N = 2560 the whole of B is live at either width).
        const long long a_block = (long long)BM * (K + p.K2) * 2;
        long long g = (16ll << 20) / (a_block > 0 ? a_block : 1);
        if (g < 8) g = 8;
        if (g > p.n_tiles_m) g = p.n_tiles_m;
        p.group_m = (int)g;
    }
    CUtensorMap ta, tb, ta2, tb2;
    int rc;
    if ((rc = br_make_tmap_2d_bf16(&ta, A, M, K, lda, BM))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tb, B, N, K, ldb, bn))) return rc;
    if (p.K2) {
        BR_CHECK_ARG(K2 % 8 == 0 && lda2 % 8 == 0 && ldb2 % 8 == 0, "gemm: K2, lda2, ldb2 must be multiples of 8");
        if ((rc = br_make_tmap_2d_bf16(&ta2, A2, M, K2, lda2, BM))) return rc;
        if ((rc = br_make_tmap_2d_bf16(&tb2, B2, N, K2, ldb2, bn))) return rc;
    } else { ta2 = ta; tb2 = tb; }
    if (masked) return launch<128, MODE_STD, true>(ta, tb, ta2, tb2, p, st);
    return wide ? launch_mode<256>(mode, ta, tb, ta2, tb2, p, st) : launch_mode<128>(mode, ta, tb, ta2, tb2, p, st);
}

}  // namespace

int br_make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) { br_set_error("cuTensorMapEncodeTiled not available from the driver"); return BR_ERR_CUDA; }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstr[1] = {ld_elems * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        br_set_error("cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu ld=%llu box_rows=%u base=%p", (int)r, (unsigned long long)rows,
                     (unsigned long long)cols, (unsigned long long)ld_elems, box_rows, base);
        return BR_ERR_CUDA;
    }
    return BR_OK;
}

extern "C" {

int br_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, void* D, int64_t ldd, int M, int N, int K,
                 const br_gemm_epilogue* e, void* stream) {
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.D = D; p.ldd = (int)ldd; p.alpha = 1.f;
    const void *A2 = nullptr, *B2 = nullptr; int64_t lda2 = 0, ldb2 = 0; int K2 = 0;
    bool masked = false;
    if (e) {
        p.bias = e->bias; p.bias_f32 = e->bias_dtype == BR_F32;
        p.residual = reinterpret_cast<const bf16*>(e->residual); p.ldr = e->ldr;
        p.alpha = e->alpha; p.act = e->act; p.out_f32 = e->out_dtype == BR_F32;
        p.row_map = e->row_map; p.aux = reinterpret_cast<bf16*>(e->aux_out); p.ld_aux = e->ld_aux;
        A2 = e->A2; B2 = e->B2; lda2 = e->lda2; ldb2 = e->ldb2; K2 = e->K2;
        BR_CHECK_ARG(!(p.act == 1 && (p.out_f32 || p.residual)), "gemm: gated-SiLU epilogue writes bf16 without residual");
        BR_CHECK_ARG(!(p.act == 1 && N % 16 != 0), "gemm: gated-SiLU epilogue needs N %% 16 == 0");
        if (e->lora_dropout) {
            int rc;
            if ((rc = br::check_drop(e->lora_dropout, "gemm"))) return rc;
            const int r = e->lora_dropout->r;
            BR_CHECK_ARG(A2 && B2 && r % 16 == 0 && r > 0 && K2 % r == 0 && e->lora_dropout->proj + K2 / r <= 8,
                         "gemm: masked LoRA segment needs A2/B2 with K2 = n_proj * r, r %% 16 == 0 (K2=%d r=%d)", K2, r);
            BR_CHECK_ARG(!p.row_map, "gemm: masked LoRA segment indexes mask rows by input row; no row_map");
            p.drop = br::drop_params(*e->lora_dropout);
            masked = true;
        }
    }
    BR_CHECK_ARG(ldd % 8 == 0 && (uintptr_t)D % 16 == 0, "gemm: D must be 16-byte aligned with ldd %% 8 == 0");
    return run_gemm(MODE_STD, A, lda, B, ldb, M, N, K, A2, lda2, B2, ldb2, K2, p, (cudaStream_t)stream, masked);
}

int64_t br_lmhead_workspace_bytes(int M, int V) {
    int nt = (V + 127) / 128;   // one (max, sum-exp) partial per 128-column tile at either tile width
    return (int64_t)M * nt * 2 * sizeof(float) + (int64_t)M * sizeof(float);
}

int br_lmhead_logprob_fwd(const void* H, int64_t ldh, const void* W, int64_t ldw, const int32_t* target, int M, int V, int K, float scale,
                          float* logp, float* lse, void* workspace, void* stream) {
    GemmParams p;
    memset(&p, 0, sizeof(p));
    int nt_max = (V + 127) / 128;
    p.alpha = scale; p.target = target;
    p.pmax = reinterpret_cast<float*>(workspace);
    p.psum = p.pmax + (int64_t)M * nt_max;
    p.tgt_logit = p.psum + (int64_t)M * nt_max;
    cudaStream_t st = (cudaStream_t)stream;
    BR_CHECK_CUDA(cudaMemsetAsync(p.tgt_logit, 0, (size_t)M * sizeof(float), st));
    int rc = run_gemm(MODE_LSE, H, ldh, W, ldw, M, V, K, nullptr, 0, nullptr, 0, 0, p, st);
    if (rc) return rc;
    const int wpb = 8;
    lse_combine_kernel<<<(M + wpb - 1) / wpb, wpb * 32, 0, st>>>(p.pmax, p.psum, p.tgt_logit, target, M, p.n_tiles_n, lse, logp);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int64_t br_lmhead_entropy_workspace_bytes(int M, int V) {
    int nt = (V + 127) / 128;   // (max, sum-exp, entropy) partials per 128-column tile
    return (int64_t)M * nt * 3 * sizeof(float) + (int64_t)M * sizeof(float);
}

int br_lmhead_logprob_entropy_fwd(const void* H, int64_t ldh, const void* W, int64_t ldw, const int32_t* target, int M, int V, int K,
                                  float scale, float* logp, float* lse, float* entropy, void* workspace, void* stream) {
    BR_CHECK_ARG(entropy, "lmhead_logprob_entropy: needs entropy");
    GemmParams p;
    memset(&p, 0, sizeof(p));
    int nt_max = (V + 127) / 128;
    p.alpha = scale; p.target = target;
    p.pmax = reinterpret_cast<float*>(workspace);
    p.psum = p.pmax + (int64_t)M * nt_max;
    p.pent = p.psum + (int64_t)M * nt_max;
    p.tgt_logit = p.pent + (int64_t)M * nt_max;
    cudaStream_t st = (cudaStream_t)stream;
    BR_CHECK_CUDA(cudaMemsetAsync(p.tgt_logit, 0, (size_t)M * sizeof(float), st));
    int rc = run_gemm(MODE_LSE_ENT, H, ldh, W, ldw, M, V, K, nullptr, 0, nullptr, 0, 0, p, st);
    if (rc) return rc;
    const int wpb = 8;
    lse_entropy_combine_kernel<<<(M + wpb - 1) / wpb, wpb * 32, 0, st>>>(p.pmax, p.psum, p.pent, p.tgt_logit, target, M, p.n_tiles_n, lse,
                                                                         logp, entropy);
    BR_CHECK_LAUNCH();
    return BR_OK;
}

int br_lmhead_dlogits(const void* H, int64_t ldh, const void* W, int64_t ldw, const int32_t* target, const float* lse, const float* gscale,
                      int M, int V, int K, float scale, void* dlogits, int64_t ldd, void* stream) {
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.alpha = scale; p.target = target; p.lse = lse; p.gscale = gscale; p.D = dlogits; p.ldd = (int)ldd;
    BR_CHECK_ARG(ldd % 8 == 0, "lmhead_dlogits: ldd %% 8");
    return run_gemm(MODE_DLOGITS, H, ldh, W, ldw, M, V, K, nullptr, 0, nullptr, 0, 0, p, (cudaStream_t)stream);
}

}  // extern "C"
