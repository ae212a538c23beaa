// Decode-time weight-streaming GEMM on wgmma (swap-AB, stream-K, persistent):  out[R, N] = X[R, K] . W[N, K]^T, R <= 32.
//
// Every decode step reads every weight byte once (SURVEY.md §8d: 8 GB / step for Qwen3-4B), so the kernel is HBM-bound and is
// built around bytes in flight, not FLOPs:
//   * swap-AB: the weight matrix is the M operand (128 output features = two m64 products), the R live rows of X are the N operand
//     (N = 16 or 32; TMA zero-fills the rows beyond R), accumulator [128 features x N] fp32 in registers;
//   * one persistent CTA per SM; a TMA producer warp keeps a 5-stage (R <= 16) or 4-stage ring of 128x64 weight tiles (16 KB each,
//     128B-swizzled) in flight (<= 101 KB of shared memory, so this kernel and its PDL successor co-reside on an SM; the successor fills its ring
//     BEFORE it waits for this kernel -- weights are constant during a rollout); one consumer warpgroup issues wgmma and runs
//     the epilogue.  (Pulling more of the chunk into L2 ahead of time was measured SLOWER: more bytes in flight only add
//     queueing delay to the small latency-critical messages -- partial tiles, counters, activations.);
//   * stream-K: the (feature tile, k block) units of the whole layer are cut into equal contiguous chunks, one per CTA, so
//     small-N layers (o_proj / down_proj: 20 feature tiles) still load all SMs evenly.  A tile finished by several CTAs
//     is reduced deterministically: every contributor writes its fp32 partial tile to its own scratch slot, the last arriver
//     (arrival counter) sums the slots in ascending CTA order and applies the epilogue -- no floating-point atomics.
// Epilogues: bf16 store, +residual, SwiGLU over (8 gate | 8 up) feature blocks, fp32 logits.
// Weight format (template parameter FP8): bf16 tiles by 2-D TMA (128B swizzle, both wgmma operands in shared memory), or e4m3 units
// (fp8_weights.cuh: 8 KB per 128x64 unit, one bulk copy, fragment order) that the consumer converts exactly to the bf16 register-A
// operand; the per-row fp32 scale multiplies the finished accumulator before the epilogue.  Half the bytes per stage buys a deeper
// ring in the same shared memory.
// PDL: the kernel is launched with programmatic stream serialization.  Kernels chained this way are NOT separated by the
// usual launch-boundary L1 invalidation, so every load of data another kernel of the chain rewrites (residual, statistics,
// scratch) goes through L2 (ld.global.cg / TMA), never through L1.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "wgmma.cuh"
#include "fp8_weights.cuh"

namespace {

constexpr int BM = 128, BK = 64, NTHREADS = 160;      // warps 0..3: wgmma + epilogue (one warpgroup), warp 4: TMA producer

struct SkParams {
    int R, N, K;
    int tiles_n, KB, units, chunk;     // units = tiles_n * KB, chunk = units per CTA
    int mode;                           // 0 bf16, 1 bf16 + residual, 2 SwiGLU blocks, 3 fp32
    void* out; long long ldo;
    const bf16* res; long long ldr;
    float* scratch;                     // [grid, 32, 128] fp32: the partial tile each contributing CTA publishes (its chunk's first segment)
    int* counters;                      // [tiles_n], zero between launches (self-resetting)
    // folded RMSNorm (decode): out[r, :] *= rsqrt(sum_i sumsq_in[i, r] / K + eps) (the norm weight is pre-multiplied into W's
    // columns); sumsq_out[(tile*4 + warp), r] = sum over that warp's 32 features of out[r, f]^2 (bf16-rounded) -- partials are
    // written, never accumulated with atomics, and summed in a fixed order by the consumer: the rollout is reproducible.
    const float* sumsq_in; int sumsq_in_n; float* sumsq_out; float eps;
    const uint8_t* wq; const float* wscale;   // FP8 weights: e4m3 units (fp8_weights.cuh) and the per-row scales
};

__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16(x)); }


template <int BNX, bool FP8 = false>
struct SL {
    static constexpr int A_BYTES = FP8 ? br::fp8w::UNIT_BYTES : BM * BK * 2;
    static constexpr int B_BYTES = BNX * BK * 2;
    static constexpr int STAGE = A_BYTES + B_BYTES;
    // <= 101 KB per CTA: this kernel and its PDL successor fit one SM (228 KB)
    static constexpr int NSTAGE = FP8 ? (BNX == 16 ? 9 : 6) : (BNX == 16 ? 5 : 4);
    static constexpr int TILE_BYTES = NSTAGE * STAGE;
    static constexpr int TR_BYTES = BM * (BNX + 1) * 4;       // accumulator transpose: one feature row per epilogue thread
    static constexpr int TOTAL = TILE_BYTES + TR_BYTES + 1024 + 1024;   // + barriers / flags / per-row rstd + alignment slack
};

// The accumulator of one 128-feature tile over `n_units` consecutive ring stages (swap-AB: the weight tile is the M operand of two
// m64nBNXk16 wgmma products, the X tile the N operand), then transposed through shared memory so that thread et holds feature et of
// the tile for every row (the layout the epilogue and the stream-K exchange work in).  Called by the consumer warpgroup (warps 0..3).
template <int BNX, int RM, bool FP8>
__device__ __forceinline__ void mma_tile(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& s, uint32_t& ph, int n_units,
                                         float* s_tr, float (&v)[RM]) {
    using L = SL<BNX, FP8>;
    const int et = threadIdx.x, warp = et >> 5, lane = et & 31;
    float acc0[BNX / 2], acc1[BNX / 2];
#pragma unroll
    for (int i = 0; i < BNX / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    for (int i = 0; i < n_units; ++i) {
        br::mbar_wait(&full_bar[s], ph);
        const uint32_t sa = br::smem_u32(smem + s * L::STAGE);
        const uint64_t bdesc = br::wg_desc_k(sa + L::A_BYTES);
        if constexpr (FP8) {
            // this thread's A fragments of the unit: 16 bytes per k16 slice (both m64 halves), converted before the first wgmma reads them
            uint32_t a[BK / 16][2][4];
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                const uint4 q = *reinterpret_cast<const uint4*>(smem + s * L::STAGE + k * 2048 + et * 16);
                br::fp8w::e4m3x4_to_bf16x2(q.x, a[k][0][0], a[k][1][0]);
                br::fp8w::e4m3x4_to_bf16x2(q.y, a[k][0][1], a[k][1][1]);
                br::fp8w::e4m3x4_to_bf16x2(q.z, a[k][0][2], a[k][1][2]);
                br::fp8w::e4m3x4_to_bf16x2(q.w, a[k][0][3], a[k][1][3]);
            }
            br::wg_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                br::wgmma_rs<BNX>(acc0, a[k][0], bdesc + 2 * k, 1);
                br::wgmma_rs<BNX>(acc1, a[k][1], bdesc + 2 * k, 1);
            }
        } else {
            br::wg_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                br::wgmma_ss<BNX>(acc0, br::wg_desc_k(sa) + 2 * k, bdesc + 2 * k, 1);
                br::wgmma_ss<BNX>(acc1, br::wg_desc_k(sa + 64 * 128) + 2 * k, bdesc + 2 * k, 1);
            }
        }
        br::wg_commit();
        br::wg_wait<0>();
        if (et == 0) br::mbar_arrive(&empty_bar[s]);
        if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
    }
    br::wg_fence_operand(acc0);
    br::wg_fence_operand(acc1);
    asm volatile("bar.sync 1, 128;" ::: "memory");                           // the previous tile's reads of s_tr are done
    const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BNX / 8; ++i)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                s_tr[(fr + 8 * hh) * (BNX + 1) + 8 * i + fc + e] = acc0[4 * i + 2 * hh + e];
                s_tr[(64 + fr + 8 * hh) * (BNX + 1) + 8 * i + fc + e] = acc1[4 * i + 2 * hh + e];
            }
    asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
    for (int r = 0; r < RM; ++r) v[r] = s_tr[et * (BNX + 1) + r];
}

// residual values of feature f for all live rows, issued as independent L2 loads (one round trip instead of R dependent ones);
// called BEFORE the accumulator wait so the latency hides under the weight stream
template <int BNX>
__device__ __forceinline__ void load_residual(const SkParams& p, int f, float (&res)[BNX]) {
    const bool on = p.mode == 1 && f < p.N;
#pragma unroll
    for (int r = 0; r < BNX; ++r) {
        res[r] = 0.f;
        if (on && r < p.R) res[r] = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(p.res) + (long long)r * p.ldr + f)));
    }
}

// per-feature epilogue: v[r] = sum for row r of feature f
template <int BNX>
__device__ __forceinline__ void apply_epilogue(const SkParams& p, int f, int lane, const float (&v)[BNX], const float (&res)[BNX], const float* s_rs, int part_row) {
    const bool f_ok = f < p.N;
    float rs[BNX];
#pragma unroll
    for (int r = 0; r < BNX; ++r) rs[r] = s_rs[r];
    if (p.mode == 2) {
        // lanes 0-7 / 16-23 hold gate features, 8-15 / 24-31 the matching up features (blocks of 16 features)
#pragma unroll
        for (int r = 0; r < BNX; ++r) {
            const float other = __shfl_down_sync(0xffffffffu, v[r], 8);
            if (r < p.R && f_ok && (lane & 8) == 0) {
                const float g = rbf(v[r] * rs[r]), u = rbf(other * rs[r]);
                const float sg = rbf(g / (1.f + __expf(-g)));
                reinterpret_cast<bf16*>(p.out)[(long long)r * p.ldo + (f >> 4) * 8 + (f & 7)] = __float2bfloat16(sg * u);
            }
        }
        return;
    }
    float sq[BNX];
#pragma unroll
    for (int r = 0; r < BNX; ++r) {
        sq[r] = 0.f;
        if (r < p.R && f_ok) {
            float x = v[r] * rs[r];
            if (p.mode == 3) reinterpret_cast<float*>(p.out)[(long long)r * p.ldo + f] = x;
            else {
                if (p.mode == 1) x = rbf(x) + res[r];
                const bf16 xb = __float2bfloat16(x);
                reinterpret_cast<bf16*>(p.out)[(long long)r * p.ldo + f] = xb;
                sq[r] = __bfloat162float(xb) * __bfloat162float(xb);
            }
        }
    }
    if (p.sumsq_out) {
#pragma unroll
        for (int r = 0; r < BNX; ++r) {
            if (r >= p.R) break;                                   // warp-uniform
            const float t = br::warp_sum(sq[r]);
            if (lane == 0) p.sumsq_out[(long long)part_row * 32 + r] = t;
        }
    }
}


// Per-row rstd of the folded RMSNorm from the producer's partial sums of squares, summed in a FIXED order (reproducible) but
// with the L2 loads spread over all 128 epilogue threads and issued in batches (a serial loop of ~80 dependent L2 round
// trips here used to cost ~30 us per GEMM).  s_part: [4][32] floats of shared scratch.  Ends with the epilogue-group barrier.
__device__ __forceinline__ void compute_row_rstd(const SkParams& p, int et, float* s_rs, float* s_part) {
    const int r = et & 31, q = et >> 5;                       // row, quarter of the partial list
    float acc = 0.f;
    if (p.sumsq_in && r < p.R) {
        const int n = p.sumsq_in_n;
        const int per = (n + 3) >> 2, lo = q * per, hi = min(n, lo + per);
        for (int i = lo; i < hi; i += 32) {                       // 32 independent L2 loads in flight: one round trip for d <= 4096
            float t[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) t[j] = (i + j < hi) ? __ldcg(p.sumsq_in + (long long)(i + j) * 32 + r) : 0.f;
#pragma unroll
            for (int j = 0; j < 32; ++j) acc += t[j];               // fixed order: reproducible
        }
    }
    s_part[q * 32 + r] = acc;
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (et < 32) {
        float rsv = 1.f;
        if (p.sumsq_in && et < p.R) rsv = rsqrtf((((s_part[et] + s_part[32 + et]) + s_part[64 + et]) + s_part[96 + et]) / (float)p.K + p.eps);
        s_rs[et] = rsv;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
}


// one weight unit (feature tile `tile`, k block `kb`; unit index u) into a ring stage: a 2-D TMA tile, or the unit's contiguous e4m3 bytes
template <int BNX, bool FP8>
__device__ __forceinline__ void load_w(uint8_t* dst, const CUtensorMap* tmW, const SkParams& p, uint64_t* bar, int u, int kb, int tile, uint64_t pol) {
    if constexpr (FP8) br::bulk_load_hint(dst, p.wq + (long long)u * SL<BNX, FP8>::A_BYTES, SL<BNX, FP8>::A_BYTES, bar, pol);
    else br::tma_load_2d_hint(dst, tmW, bar, kb * BK, tile * BM, pol);
}


// BNX: wgmma N (rows of X the tensor core sees, zero-filled beyond R); RM: rows the epilogue code is generated for (R <= RM <= BNX).
// The epilogue runs once per CTA per launch -- straight-line, instruction-fetch-bound code -- so the common R <= 8 decode batch gets its
// own half-size instantiation.  Warps 0..3: wgmma + epilogue (one feature row per thread), warp 4: TMA producer.
template <int BNX, int RM, bool FP8>
__global__ void __launch_bounds__(NTHREADS, 1)
skinny_tc5_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
                  const __grid_constant__ SkParams p) {      // read in place by the helpers (const SkParams&): no register copy
    using L = SL<BNX, FP8>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* s_tr = reinterpret_cast<float*>(smem + L::TILE_BYTES);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::TILE_BYTES + L::TR_BYTES);
    uint64_t* empty_bar = full_bar + L::NSTAGE;
    float* s_rs = reinterpret_cast<float*>(empty_bar + L::NSTAGE);   // [32] per-row rstd of the folded RMSNorm (+ [4][32] scratch)

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int u_lo = blockIdx.x * p.chunk;
    const int u_hi = min(p.units, u_lo + p.chunk);

    br::launch_dependents();
    if (threadIdx.x == 0) {
        br::tma_prefetch_desc(&tmW);
        br::tma_prefetch_desc(&tmX);
        for (int s = 0; s < L::NSTAGE; ++s) { br::mbar_init(&full_bar[s], 1); br::mbar_init(&empty_bar[s], 1); }
        br::mbar_fence_init();
    }
    __syncthreads();
    const int n_units = u_hi - u_lo;

    if (warp == 4) {
        if (lane == 0) {
            // The weights are constant during the rollout: fill the whole ring with weight tiles BEFORE waiting for the
            // previous kernel (PDL), so the HBM stream of this layer overlaps the tail of the previous kernel.
            const int n_pre = min(L::NSTAGE, n_units);
            // weight tiles are read once per token step: evict-first in L2, so the small latency-critical buffers (activations,
            // partial tiles, statistics, tables) stay resident
            const uint64_t pol = br::make_policy_evict_first();
            for (int i = 0; i < n_pre; ++i) {
                const int u = u_lo + i, tile = u / p.KB, kb = u - tile * p.KB;
                br::mbar_expect_tx(&full_bar[i], L::STAGE);
                load_w<BNX, FP8>(smem + i * L::STAGE, &tmW, p, &full_bar[i], u, kb, tile, pol);
            }
            br::grid_dep_wait();
            for (int i = 0; i < n_pre; ++i) {
                const int u = u_lo + i, tile = u / p.KB, kb = u - tile * p.KB;
                br::tma_load_2d(smem + i * L::STAGE + L::A_BYTES, &tmX, &full_bar[i], kb * BK, 0);
            }
            int s = n_pre % L::NSTAGE; uint32_t ph = (n_pre == L::NSTAGE) ? 1u : 0u;
            for (int u = u_lo + n_pre; u < u_hi; ++u) {
                const int tile = u / p.KB, kb = u - tile * p.KB;
                br::mbar_wait(&empty_bar[s], ph ^ 1);
                uint8_t* sa = smem + s * L::STAGE;
                br::mbar_expect_tx(&full_bar[s], L::STAGE);
                load_w<BNX, FP8>(sa, &tmW, p, &full_bar[s], u, kb, tile, pol);
                br::tma_load_2d(sa + L::A_BYTES, &tmX, &full_bar[s], kb * BK, 0);
                if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
            }
        }
    } else {
        const int lane_grp = warp & 3;
        const int et = threadIdx.x;                               // 0..127 within the consumer warpgroup
        br::grid_dep_wait();                                      // everything below touches data shared with earlier kernels
        compute_row_rstd(p, et, s_rs, s_rs + 32);
        int s = 0; uint32_t ph = 0;
        int u = u_lo;
        while (u < u_hi) {
            const int tile = u / p.KB;
            const int seg_end = min(u_hi, (tile + 1) * p.KB);
            const bool whole = (u == tile * p.KB) && (seg_end == (tile + 1) * p.KB);
            const int f = tile * BM + lane_grp * 32 + lane;
            const int part_row = tile * 4 + lane_grp;
            float res[RM];
            load_residual<RM>(p, f, res);                        // in flight while the accumulator is still being produced
            float wsc = 0.f;
            if constexpr (FP8) wsc = f < p.N ? __ldcg(p.wscale + f) : 0.f;
            float v[RM];
            mma_tile<BNX, RM, FP8>(smem, full_bar, empty_bar, s, ph, seg_end - u, s_tr, v);
            if constexpr (FP8) {
                if (whole) {                                      // the per-row weight scale, once on the finished sum (stream-K: below)
#pragma unroll
                    for (int r = 0; r < RM; ++r) v[r] *= wsc;
                }
            }
            if (whole) {
                apply_epilogue<RM>(p, f, lane, v, res, s_rs, part_row);
            } else {
                // Deterministic stream-K exchange.  A tile that spans several CTAs is finished by the FIRST of them (lowest index):
                // for that CTA the tile is the last segment of its chunk, so it has nothing else left to do, while every other
                // contributor meets the tile at the START of its chunk and publishes early.  Contributors store their fp32 partial
                // tile to their scratch slot and signal with one release-reduction per warp (no CTA barrier, no fence, no returning
                // atomic); the reducer acquires the counter, gathers all partials in ONE batch of independent L2 loads and adds them
                // to its own registers in ascending CTA order -- no floating-point atomics, bit-reproducible.
                const int first_c = (tile * p.KB) / p.chunk, last_c = ((tile + 1) * p.KB - 1) / p.chunk;
                if ((int)blockIdx.x != first_c) {
                    float* mine = p.scratch + (long long)blockIdx.x * 32 * BM + lane_grp * 32 + lane;
    #pragma unroll
                    for (int r = 0; r < RM; ++r)
                        if (r < p.R) __stcg(mine + r * BM, v[r]);
                    __syncwarp();
                    if (lane == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p.counters + tile) : "memory");
                } else {
                    if (et == 0) {
                        const unsigned want = 4u * (unsigned)(last_c - first_c);
                        unsigned seen;
                        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(p.counters + tile) : "memory"); } while (seen < want);
                        p.counters[tile] = 0;                                    // nobody touches it again before the next launch
                    }
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    for (int c0 = first_c + 1; c0 <= last_c; c0 += 8) {          // 8 contributors x 8 rows of loads in flight
    #pragma unroll
                        for (int r0 = 0; r0 < RM; r0 += 8) {
                            if (r0 >= p.R) break;                                // warp-uniform
                            float t[8][8];
    #pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                const float* src = p.scratch + (long long)(c0 + j) * 32 * BM + lane_grp * 32 + lane;
    #pragma unroll
                                for (int r = 0; r < 8; ++r) t[j][r] = (c0 + j <= last_c && r0 + r < p.R) ? __ldcg(src + (r0 + r) * BM) : 0.f;
                            }
    #pragma unroll
                            for (int j = 0; j < 8; ++j)
    #pragma unroll
                                for (int r = 0; r < 8; ++r) v[r0 + r] += t[j][r];            // ascending CTA order: deterministic
                        }
                    }
                    if constexpr (FP8) {
#pragma unroll
                        for (int r = 0; r < RM; ++r) v[r] *= wsc;
                    }
                    apply_epilogue<RM>(p, f, lane, v, res, s_rs, part_row);
                }
            }
            u = seg_end;
        }
    }
}

template <int BNX, int RM, bool FP8>
int launch(const CUtensorMap& tw, const CUtensorMap& tx, const SkParams& p, int grid, cudaStream_t st) {
    using L = SL<BNX, FP8>;
    auto kern = skinny_tc5_kernel<BNX, RM, FP8>;
    static bool done = false;
    if (!done) {
        BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
        done = true;
    }
    BR_CHECK_CUDA(br_launch_pdl(kern, dim3(grid), dim3(NTHREADS), (size_t)L::TOTAL, st, tw, tx, p));
    return BR_OK;
}

// shared host side of br_skinny_gemm / br_skinny_gemm_fp8 (w_scale != NULL: W is the e4m3 buffer of br_quantize_rows_e4m3)
int skinny_run(const void* X, int64_t ldx, const void* W, int64_t ldw, const float* w_scale, void* out, int64_t ldo, int R, int N, int K,
               int mode, const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n, float* sumsq_out, float eps,
               void* stream) {
    const bool fp8 = w_scale != nullptr;
    BR_CHECK_ARG(R >= 1 && R <= 32, "skinny_gemm: R=%d must be in [1, 32]", R);
    BR_CHECK_ARG(N % 16 == 0 && K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "skinny_gemm: N %% 16, K %% 8, ld %% 8 (N=%d K=%d)", N, K);
    BR_CHECK_ARG(mode >= 0 && mode <= 3 && !(mode == 1 && !residual), "skinny_gemm: bad mode %d", mode);
    BR_CHECK_ARG(scratch != nullptr, "skinny_gemm: scratch (br_skinny_scratch_bytes, zero-initialised once) is required");
    if (fp8) {
        BR_CHECK_ARG(K % 16 == 0 && ldw == K, "skinny_gemm_fp8: K must be a multiple of 16 and ldw == K (the quantized layout; N=%d K=%d ldw=%lld)",
                     N, K, (long long)ldw);
        BR_CHECK_ARG(W != nullptr && ((uintptr_t)W & 15) == 0, "skinny_gemm_fp8: W must be the 16-byte aligned buffer of br_quantize_rows_e4m3");
    }
    SkParams p;
    p.R = R; p.N = N; p.K = K; p.mode = mode; p.out = out; p.ldo = ldo; p.res = (const bf16*)residual; p.ldr = ldr;
    p.scratch = (float*)scratch; p.counters = (int*)((float*)scratch + (int64_t)br_num_sms() * 32 * BM);
    p.sumsq_in = sumsq_in; p.sumsq_in_n = sumsq_in_n; p.sumsq_out = sumsq_out; p.eps = eps;
    p.wq = fp8 ? (const uint8_t*)W : nullptr; p.wscale = w_scale;
    BR_CHECK_ARG(!(sumsq_out && mode >= 2), "skinny_gemm: sumsq_out only with bf16 outputs (mode 0/1)");
    p.tiles_n = (N + BM - 1) / BM; p.KB = (K + BK - 1) / BK; p.units = p.tiles_n * p.KB;
    int grid = p.units < br_num_sms() ? p.units : br_num_sms();
    p.chunk = (p.units + grid - 1) / grid;
    grid = (p.units + p.chunk - 1) / p.chunk;
    const int BNX = R <= 16 ? 16 : 32;
    CUtensorMap tw, tx;
    int rc;
    if ((rc = br_make_tmap_2d_bf16(&tx, X, R, K, ldx, BNX))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (fp8) {                                                    // the weights come by bulk copy: no weight tensor map
        if (R <= 8) return launch<16, 8, true>(tx, tx, p, grid, st);
        return BNX == 16 ? launch<16, 16, true>(tx, tx, p, grid, st) : launch<32, 32, true>(tx, tx, p, grid, st);
    }
    if ((rc = br_make_tmap_2d_bf16(&tw, W, N, K, ldw, BM))) return rc;
    if (R <= 8) return launch<16, 8, false>(tw, tx, p, grid, st);
    return BNX == 16 ? launch<16, 16, false>(tw, tx, p, grid, st) : launch<32, 32, false>(tw, tx, p, grid, st);
}

}  // namespace

extern "C" {

int64_t br_skinny_scratch_bytes(int max_N) {
    // partial tiles [n_sms, 32, 128] fp32 | one arrival counter per 128-feature tile
    return (int64_t)br_num_sms() * 32 * BM * sizeof(float) + (int64_t)(max_N / BM + 2) * sizeof(int);
}

int br_skinny_gemm(const void* X, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, int R, int N, int K, int mode,
                   const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n, float* sumsq_out, float eps,
                   void* stream) {
    return skinny_run(X, ldx, W, ldw, nullptr, out, ldo, R, N, K, mode, residual, ldr, scratch, sumsq_in, sumsq_in_n, sumsq_out, eps, stream);
}

int br_skinny_gemm_fp8(const void* X, int64_t ldx, const void* W, int64_t ldw, const float* w_scale, void* out, int64_t ldo, int R, int N,
                       int K, int mode, const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n,
                       float* sumsq_out, float eps, void* stream) {
    BR_CHECK_ARG(w_scale != nullptr, "skinny_gemm_fp8: w_scale (one fp32 scale per row of W) is required");
    return skinny_run(X, ldx, W, ldw, w_scale, out, ldo, R, N, K, mode, residual, ldr, scratch, sumsq_in, sumsq_in_n, sumsq_out, eps, stream);
}

}  // extern "C"
