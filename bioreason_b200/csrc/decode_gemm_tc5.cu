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
// PDL: the kernel is launched with programmatic stream serialization.  Kernels chained this way are NOT separated by the
// usual launch-boundary L1 invalidation, so every load of data another kernel of the chain rewrites (residual, statistics,
// scratch) goes through L2 (ld.global.cg / TMA), never through L1.
#include "br_common.cuh"
#include "../../include/bioreason_b200.h"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128, BK = 64, NTHREADS = 160;      // warps 0..3: wgmma + epilogue (one warpgroup), warp 4: TMA producer

struct SkParams {
    int R, N, K;
    int tiles_n, KB, units, chunk;     // units = tiles_n * KB, chunk = units per CTA
    int mode;                           // 0 bf16, 1 bf16 + residual, 2 SwiGLU blocks, 3 fp32
    void* out; long long ldo;
    const bf16* res; long long ldr;
    float* scratch;                     // [grid, 2, BNX, 128] fp32 partial tiles (slot 0: CTA's first tile, 1: its last tile)
    int* counters;                      // [tiles_n], zero between launches (self-resetting)
    // folded RMSNorm (decode): out[r, :] *= rsqrt(sum_i sumsq_in[i, r] / K + eps) (the norm weight is pre-multiplied into W's
    // columns); sumsq_out[(tile*4 + warp), r] = sum over that warp's 32 features of out[r, f]^2 (bf16-rounded) -- partials are
    // written, never accumulated with atomics, and summed in a fixed order by the consumer: the rollout is reproducible.
    const float* sumsq_in; int sumsq_in_n; float* sumsq_out; float eps;
    long long* dbg; int dbg_slot;       // optional %globaltimer stamps [slot][cta][8] (profiling aid)
    br::L2Prefetch pf; int pf_on;       // L2 staging of a later GEMM's weights (see br_common.cuh)
    int* gate_counter; const int* gate_epoch; int gate_base, gate_per_step, gate_wait, gate_signal;   // stream gate (see br_stream_gate)
    int w_evict_first;                  // weight tiles are read once per token step: mark them evict-first in L2 so the small
                                        // latency-critical buffers (activations, partial tiles, statistics, tables) stay resident
};

__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16(x)); }


template <int BNX>
struct SL {
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BNX * BK * 2;
    static constexpr int STAGE = A_BYTES + B_BYTES;
    static constexpr int NSTAGE = BNX == 16 ? 5 : 4;         // <= 101 KB per CTA: this kernel and its PDL successor fit one SM (228 KB)
    static constexpr int TILE_BYTES = NSTAGE * STAGE;
    static constexpr int TR_BYTES = BM * (BNX + 1) * 4;       // accumulator transpose: one feature row per epilogue thread
    static constexpr int TOTAL = TILE_BYTES + TR_BYTES + 1024 + 1024;   // + barriers / flags / per-row rstd + alignment slack
};

// The accumulator of one 128-feature tile over `n_units` consecutive ring stages (swap-AB: the weight tile is the M operand of two
// m64nBNXk16 wgmma products, the X tile the N operand), then transposed through shared memory so that thread et holds feature et of
// the tile for every row (the layout the epilogue and the stream-K exchange work in).  Called by the consumer warpgroup (warps 0..3).
template <int BNX, int RM>
__device__ __forceinline__ void mma_tile(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& s, uint32_t& ph, int n_units,
                                         int* signal_counter, float* s_tr, float (&v)[RM]) {
    using L = SL<BNX>;
    const int et = threadIdx.x, warp = et >> 5, lane = et & 31;
    float acc0[BNX / 2], acc1[BNX / 2];
#pragma unroll
    for (int i = 0; i < BNX / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    for (int i = 0; i < n_units; ++i) {
        br::mbar_wait(&full_bar[s], ph);
        if (i == n_units - 1 && signal_counter && et == 0)                    // every weight tile of this CTA is on chip
            asm volatile("red.relaxed.gpu.global.add.s32 [%0], 1;" ::"l"(signal_counter) : "memory");
        const uint32_t sa = br::smem_u32(smem + s * L::STAGE);
        const uint64_t bdesc = br::wg_desc_k(sa + L::A_BYTES);
        br::wg_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
            br::wgmma_ss<BNX>(acc0, br::wg_desc_k(sa) + 2 * k, bdesc + 2 * k, 1);
            br::wgmma_ss<BNX>(acc1, br::wg_desc_k(sa + 64 * 128) + 2 * k, bdesc + 2 * k, 1);
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

__device__ __forceinline__ long long gtime_sk() { long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define SKSTAMP(k) do { if (p.dbg && (threadIdx.x == 0)) p.dbg[((long long)p.dbg_slot * 160 + blockIdx.x) * 8 + (k)] = gtime_sk(); } while (0)


// BNX: wgmma N (rows of X the tensor core sees, zero-filled beyond R); RM: rows the epilogue code is generated for (R <= RM <= BNX).
// The epilogue runs once per CTA per launch -- straight-line, instruction-fetch-bound code -- so the common R <= 8 decode batch gets its
// own half-size instantiation.  Warps 0..3: wgmma + epilogue (one feature row per thread), warp 4: TMA producer.
template <int BNX, int RM>
__global__ void __launch_bounds__(NTHREADS, 1)
skinny_tc5_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmP,
                  const SkParams p) {
    using L = SL<BNX>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* s_tr = reinterpret_cast<float*>(smem + L::TILE_BYTES);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::TILE_BYTES + L::TR_BYTES);
    uint64_t* empty_bar = full_bar + L::NSTAGE;
    int* s_flag = reinterpret_cast<int*>(empty_bar + L::NSTAGE);
    float* s_rs = reinterpret_cast<float*>(s_flag + 2);       // [32] per-row rstd of the folded RMSNorm (+ [4][32] scratch)

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int u_lo = blockIdx.x * p.chunk;
    const int u_hi = min(p.units, u_lo + p.chunk);

    br::launch_dependents();
    SKSTAMP(0);
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
            const uint64_t pol = br::make_policy_evict_first();
            if (p.gate_counter && p.gate_wait >= 0) {             // start the early loads under the previous GEMM's exchange tail, not under its stream
                const int target = (__ldcg(p.gate_epoch) - p.gate_base) * p.gate_per_step + p.gate_wait;
                for (int it = 0; it < 32; ++it) {                 // bounded: the gate is a timing hint
                    int seen;
                    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(p.gate_counter) : "memory");
                    if (seen >= target) break;
                }
            }
            auto load_w = [&](void* dst, uint64_t* bar, int c0, int c1) {
                if (p.w_evict_first) br::tma_load_2d_hint(dst, &tmW, bar, c0, c1, pol);
                else br::tma_load_2d(dst, &tmW, bar, c0, c1);
            };
            for (int i = 0; i < n_pre; ++i) {
                const int u = u_lo + i, tile = u / p.KB, kb = u - tile * p.KB;
                br::mbar_expect_tx(&full_bar[i], L::STAGE);
                load_w(smem + i * L::STAGE, &full_bar[i], kb * BK, tile * BM);
            }
            if (p.pf_on) br::l2_prefetch_issue(&tmP, p.pf, blockIdx.x, gridDim.x);     // a LATER GEMM's tiles -> L2 (HBM is otherwise idle here)
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
                load_w(sa, &full_bar[s], kb * BK, tile * BM);
                br::tma_load_2d(sa + L::A_BYTES, &tmX, &full_bar[s], kb * BK, 0);
                if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
            }
        }
    } else {
        const int lane_grp = warp & 3;
        const int et = threadIdx.x;                               // 0..127 within the consumer warpgroup
        SKSTAMP(2);                                               // barriers initialised
        br::grid_dep_wait();                                      // everything below touches data shared with earlier kernels
        SKSTAMP(1);
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
            float v[RM];
            mma_tile<BNX, RM>(smem, full_bar, empty_bar, s, ph, seg_end - u, (seg_end == u_hi && p.gate_counter && p.gate_signal) ? p.gate_counter : nullptr,
                              s_tr, v);
            if (u == u_lo) SKSTAMP(3);
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
                    float* mine = p.scratch + ((long long)blockIdx.x * 2 * BNX) * BM + lane_grp * 32 + lane;   // slot 0: the CTA's first tile
    #pragma unroll
                    for (int r = 0; r < RM; ++r)
                        if (r < p.R) __stcg(mine + r * BM, v[r]);
                    __syncwarp();
                    if (lane == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p.counters + tile) : "memory");
                    if (seg_end == u_hi) SKSTAMP(4);
                } else {
                    if (et == 0) {
                        const unsigned want = 4u * (unsigned)(last_c - first_c);
                        unsigned seen;
                        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(p.counters + tile) : "memory"); } while (seen < want);
                        p.counters[tile] = 0;                                    // nobody touches it again before the next launch
                    }
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    SKSTAMP(4);
                    for (int c0 = first_c + 1; c0 <= last_c; c0 += 8) {          // 8 contributors x 8 rows of loads in flight
    #pragma unroll
                        for (int r0 = 0; r0 < RM; r0 += 8) {
                            if (r0 >= p.R) break;                                // warp-uniform
                            float t[8][8];
    #pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                const float* src = p.scratch + ((long long)(c0 + j) * 2 * BNX) * BM + lane_grp * 32 + lane;
    #pragma unroll
                                for (int r = 0; r < 8; ++r) t[j][r] = (c0 + j <= last_c && r0 + r < p.R) ? __ldcg(src + (r0 + r) * BM) : 0.f;
                            }
    #pragma unroll
                            for (int j = 0; j < 8; ++j)
    #pragma unroll
                                for (int r = 0; r < 8; ++r) v[r0 + r] += t[j][r];            // ascending CTA order: deterministic
                        }
                    }
                    SKSTAMP(5);
                    apply_epilogue<RM>(p, f, lane, v, res, s_rs, part_row);
                    SKSTAMP(6);
                }
            }
            u = seg_end;
        }
        SKSTAMP(7);
    }
}

template <int BNX, int RM>
int launch(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& tp, const SkParams& p, int grid, cudaStream_t st) {
    using L = SL<BNX>;
    auto kern = skinny_tc5_kernel<BNX, RM>;
    static bool done = false;
    if (!done) {
        BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
        done = true;
    }
    BR_CHECK_CUDA(br_launch_pdl(kern, dim3(grid), dim3(NTHREADS), (size_t)L::TOTAL, st, tw, tx, tp, p));
    return BR_OK;
}


// ================================================================================================================
// Multi-phase persistent variant: up to 4 dependent GEMMs (o_proj -> gate/up -> down_proj -> next layer's qkv, or
// ... -> lm_head) in ONE launch.  Phases are separated by a grid-wide barrier instead of a kernel boundary; the weight
// producer is not gated by the barrier, so while the CTAs synchronise (and while the last tiles of a phase are reduced)
// the ring already fills with the next phase's weights -- the HBM stream does not stop at phase boundaries.  A second
// producer thread loads the activation tiles and is the only one that waits for "phase inputs ready".
// ================================================================================================================
constexpr int CHAIN_MAX = 4;
constexpr int CHAIN_THREADS = 192;           // warps 0-3: wgmma + epilogue, 4: W producer, 5: X producer

struct ChainPhase { CUtensorMap tmW; CUtensorMap tmX; SkParams p; };
struct ChainParams { ChainPhase ph[CHAIN_MAX]; int n_phases; int* gbar; long long* dbg; };
__device__ __forceinline__ long long gtime() { long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define CSTAMP(k) do { if (cp.dbg && et == 0) cp.dbg[(long long)blockIdx.x * 32 + (k)] = gtime(); } while (0)

template <int BNX>
__global__ void __launch_bounds__(CHAIN_THREADS, 1) skinny_chain_kernel(const __grid_constant__ ChainParams cp) {
    using L = SL<BNX>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* s_tr = reinterpret_cast<float*>(smem + L::TILE_BYTES);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::TILE_BYTES + L::TR_BYTES);
    uint64_t* empty_bar = full_bar + L::NSTAGE;
    int* s_flag = reinterpret_cast<int*>(empty_bar + L::NSTAGE);
    volatile int* s_ready = reinterpret_cast<volatile int*>(s_flag + 1);      // number of grid barriers this CTA has passed
    float* s_rs = reinterpret_cast<float*>(s_flag + 2);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nph = cp.n_phases;

    br::launch_dependents();
    if (threadIdx.x == 0) {
        for (int i = 0; i < nph; ++i) { br::tma_prefetch_desc(&cp.ph[i].tmW); br::tma_prefetch_desc(&cp.ph[i].tmX); }
        // full: the W producer's expect_tx covers both halves of a stage (the X producer's load completes the same count);
        // empty: released by the consumer warpgroup, awaited by both producers
        for (int s = 0; s < L::NSTAGE; ++s) { br::mbar_init(&full_bar[s], 1); br::mbar_init(&empty_bar[s], 1); }
        br::mbar_fence_init();
        *s_ready = 0;
    }
    __syncthreads();

    if (warp == 4) {
        // ---------------- weight producer: never waits for other kernels or phases (weights are constant) ----------------
        if (lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int pi = 0; pi < nph; ++pi) {
                const SkParams& p = cp.ph[pi].p;
                const int u_lo = blockIdx.x * p.chunk, u_hi = min(p.units, u_lo + p.chunk);
                for (int u = u_lo; u < u_hi; ++u) {
                    const int tile = u / p.KB, kb = u - tile * p.KB;
                    br::mbar_wait(&empty_bar[s], ph ^ 1);
                    br::mbar_expect_tx(&full_bar[s], L::STAGE);
                    br::tma_load_2d(smem + s * L::STAGE, &cp.ph[pi].tmW, &full_bar[s], kb * BK, tile * BM);
                    if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
                }
            }
        }
    } else if (warp == 5) {
        // ---------------- activation producer: gated by "inputs of phase pi are complete" ----------------
        if (lane == 0) {
            br::grid_dep_wait();
            int s = 0; uint32_t ph = 0;
            for (int pi = 0; pi < nph; ++pi) {
                const SkParams& p = cp.ph[pi].p;
                const int u_lo = blockIdx.x * p.chunk, u_hi = min(p.units, u_lo + p.chunk);
                if (u_lo < u_hi) while (*s_ready < pi) __nanosleep(32);
                for (int u = u_lo; u < u_hi; ++u) {
                    const int tile = u / p.KB, kb = u - tile * p.KB;
                    br::mbar_wait(&empty_bar[s], ph ^ 1);
                    br::tma_load_2d(smem + s * L::STAGE + L::A_BYTES, &cp.ph[pi].tmX, &full_bar[s], kb * BK, 0);
                    if (++s == L::NSTAGE) { s = 0; ph ^= 1; }
                }
            }
        }
    } else {
        // ---------------- consumer warpgroup (warps 0..3): wgmma + epilogue ----------------
        const int lane_grp = warp & 3;
        const int et = threadIdx.x;
        CSTAMP(0);
        br::grid_dep_wait();
        CSTAMP(1);
        int s = 0; uint32_t ph = 0;
        for (int pi = 0; pi < nph; ++pi) {
            const SkParams& p = cp.ph[pi].p;
            const int u_lo = blockIdx.x * p.chunk, u_hi = min(p.units, u_lo + p.chunk);
            CSTAMP(2 + pi * 6);
            compute_row_rstd(p, et, s_rs, s_rs + 32);      // inputs complete: barrier pi-1 passed
            int u = u_lo;
            while (u < u_hi) {
                const int tile = u / p.KB;
                const int seg_end = min(u_hi, (tile + 1) * p.KB);
                const bool whole = (u == tile * p.KB) && (seg_end == (tile + 1) * p.KB);
                float v[BNX];
                mma_tile<BNX, BNX>(smem, full_bar, empty_bar, s, ph, seg_end - u, nullptr, s_tr, v);
                if (u == u_lo) CSTAMP(3 + pi * 6);
                const int f = tile * BM + lane_grp * 32 + lane;
                const int part_row = tile * 4 + lane_grp;
                float res[BNX];
                load_residual<BNX>(p, f, res);
                if (whole) {
                    apply_epilogue<BNX>(p, f, lane, v, res, s_rs, part_row);
                } else {
                    const int first_c = (tile * p.KB) / p.chunk, last_c = ((tile + 1) * p.KB - 1) / p.chunk;
                    const int my_slot = (tile == u_lo / p.KB) ? 0 : 1;
                    float* mine = p.scratch + (((long long)blockIdx.x * 2 + my_slot) * BNX) * BM + lane_grp * 32 + lane;
#pragma unroll
                    for (int r = 0; r < BNX; ++r)
                        if (r < p.R) __stcg(mine + r * BM, v[r]);
                    __threadfence();
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (et == 0) *s_flag = (atomicAdd(p.counters + tile, 1) == last_c - first_c);
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (*s_flag) {
                        __threadfence();
#pragma unroll
                        for (int r = 0; r < BNX; ++r) v[r] = 0.f;
                        for (int c0 = first_c; c0 <= last_c; c0 += 4) {
                            float t[4][BNX];
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const int c = c0 + j;
                                const int slot = (tile == (c * p.chunk) / p.KB) ? 0 : 1;
                                const float* src = p.scratch + (((long long)c * 2 + slot) * BNX) * BM + lane_grp * 32 + lane;
#pragma unroll
                                for (int r = 0; r < BNX; ++r) t[j][r] = (c <= last_c && r < p.R) ? __ldcg(src + r * BM) : 0.f;
                            }
#pragma unroll
                            for (int j = 0; j < 4; ++j)
#pragma unroll
                                for (int r = 0; r < BNX; ++r) v[r] += t[j][r];
                        }
                        if (et == 0) p.counters[tile] = 0;
                        apply_epilogue<BNX>(p, f, lane, v, res, s_rs, part_row);
                    }
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                }
                u = seg_end;
            }
            CSTAMP(4 + pi * 6);
            if (pi + 1 < nph) {
                // grid barrier: every CTA's outputs of phase pi are globally visible before anyone loads them as phase pi+1 inputs
                __threadfence();
                asm volatile("bar.sync 1, 128;" ::: "memory");
                CSTAMP(5 + pi * 6);
                if (et == 0) {
                    atomicAdd(cp.gbar, 1);
                    const int target = (pi + 1) * (int)gridDim.x;
                    int seen;
                    do { asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(cp.gbar) : "memory"); } while (seen < target);
                    *s_ready = pi + 1;
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");
                CSTAMP(6 + pi * 6);
            }
        }
        // the last CTA to finish re-zeros the barrier words for the next launch (everyone else has left the barrier code)
        if (et == 0 && nph > 1) {
            if (atomicAdd(cp.gbar + 1, 1) == (int)gridDim.x - 1) { cp.gbar[0] = 0; cp.gbar[1] = 0; __threadfence(); }
        }
    }
}

template <int BNX>
int launch_chain(const ChainParams& cp, int grid, cudaStream_t st) {
    using L = SL<BNX>;
    auto kern = skinny_chain_kernel<BNX>;
    static bool done = false;
    if (!done) { BR_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL)); done = true; }
    BR_CHECK_CUDA(br_launch_pdl(kern, dim3(grid), dim3(CHAIN_THREADS), (size_t)L::TOTAL, st, cp));
    return BR_OK;
}

}  // namespace

static long long* g_sk_dbg = nullptr;
static int g_sk_dbg_slot = 0;

int br_make_l2_prefetch(const br_l2_prefetch* spec, CUtensorMap* tmap, int* KB, int* units, int* chunk, int* n_chunks, int* a, int* b) {
    BR_CHECK_ARG(spec->N % 16 == 0 && spec->K % 8 == 0 && spec->ldw % 8 == 0 && spec->unit_lo >= 0, "l2_prefetch: bad weight shape");
    const int tiles_n = (spec->N + BM - 1) / BM;
    *KB = (spec->K + BK - 1) / BK; *units = tiles_n * *KB;
    int grid = *units < br_num_sms() ? *units : br_num_sms();
    *chunk = (*units + grid - 1) / grid;
    *n_chunks = (*units + *chunk - 1) / *chunk;
    *a = spec->unit_lo; *b = spec->unit_hi;
    return br_make_tmap_2d_bf16(tmap, spec->W, spec->N, spec->K, spec->ldw, BM);
}

extern "C" {

int64_t br_skinny_scratch_bytes(int max_N) {
    // partial tiles [n_sms, 2, 32, 128] fp32 | grid-barrier word (16 ints) | one arrival counter per 128-feature tile
    return (int64_t)br_num_sms() * 2 * 32 * BM * sizeof(float) + 16 * sizeof(int) + (int64_t)(max_N / BM + 2) * sizeof(int);
}

int br_skinny_gemm(const void* X, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, int R, int N, int K, int mode,
                   const void* residual, int64_t ldr, void* scratch, void* stream) {
    return br_skinny_gemm_ex(X, ldx, W, ldw, out, ldo, R, N, K, mode, residual, ldr, scratch, nullptr, 0, nullptr, 0.f, stream);
}

int br_skinny_gemm_ex(const void* X, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, int R, int N, int K, int mode,
                      const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n, float* sumsq_out, float eps,
                      void* stream) {
    return br_skinny_gemm_pf(X, ldx, W, ldw, out, ldo, R, N, K, mode, residual, ldr, scratch, sumsq_in, sumsq_in_n, sumsq_out, eps, nullptr, stream);
}

int br_skinny_grid(int N, int K) {
    const int units = ((N + BM - 1) / BM) * ((K + BK - 1) / BK);
    int grid = units < br_num_sms() ? units : br_num_sms();
    const int chunk = (units + grid - 1) / grid;
    return (units + chunk - 1) / chunk;
}

int br_skinny_gemm_pf(const void* X, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, int R, int N, int K, int mode,
                      const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n, float* sumsq_out, float eps,
                      const br_l2_prefetch* prefetch, void* stream) {
    return br_skinny_gemm_gated(X, ldx, W, ldw, out, ldo, R, N, K, mode, residual, ldr, scratch, sumsq_in, sumsq_in_n, sumsq_out, eps, prefetch, nullptr, stream);
}

int br_skinny_gemm_gated(const void* X, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, int R, int N, int K, int mode,
                         const void* residual, int64_t ldr, void* scratch, const float* sumsq_in, int sumsq_in_n, float* sumsq_out, float eps,
                         const br_l2_prefetch* prefetch, const br_stream_gate* gate, void* stream) {
    BR_CHECK_ARG(R >= 1 && R <= 32, "skinny_gemm: R=%d must be in [1, 32]", R);
    BR_CHECK_ARG(N % 16 == 0 && K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "skinny_gemm: N %% 16, K %% 8, ld %% 8 (N=%d K=%d)", N, K);
    BR_CHECK_ARG(mode >= 0 && mode <= 3 && !(mode == 1 && !residual), "skinny_gemm: bad mode %d", mode);
    BR_CHECK_ARG(scratch != nullptr, "skinny_gemm: scratch (br_skinny_scratch_bytes, zero-initialised once) is required");
    SkParams p;
    p.R = R; p.N = N; p.K = K; p.mode = mode; p.out = out; p.ldo = ldo; p.res = (const bf16*)residual; p.ldr = ldr;
    p.scratch = (float*)scratch; p.counters = (int*)((float*)scratch + (int64_t)br_num_sms() * 2 * 32 * BM) + 16;
    p.sumsq_in = sumsq_in; p.sumsq_in_n = sumsq_in_n; p.sumsq_out = sumsq_out; p.eps = eps;
    BR_CHECK_ARG(!(sumsq_out && mode >= 2), "skinny_gemm: sumsq_out only with bf16 outputs (mode 0/1)");
    p.dbg = g_sk_dbg; p.dbg_slot = g_sk_dbg ? g_sk_dbg_slot++ : 0;
    p.gate_counter = nullptr; p.gate_epoch = nullptr; p.gate_base = p.gate_per_step = p.gate_signal = 0; p.gate_wait = -1;
    if (gate && gate->counter) {
        BR_CHECK_ARG(gate->epoch != nullptr && gate->per_step >= 0, "skinny_gemm: stream gate needs the epoch counter");
        p.gate_counter = gate->counter; p.gate_epoch = gate->epoch; p.gate_base = gate->epoch_base; p.gate_per_step = gate->per_step;
        p.gate_wait = gate->wait_prefix; p.gate_signal = gate->signal;
    }
    { const char* e = getenv("BR_SKINNY_EVICT_FIRST"); p.w_evict_first = e ? atoi(e) : 1; }
    p.tiles_n = (N + BM - 1) / BM; p.KB = (K + BK - 1) / BK; p.units = p.tiles_n * p.KB;
    int grid = p.units < br_num_sms() ? p.units : br_num_sms();
    p.chunk = (p.units + grid - 1) / grid;
    grid = (p.units + p.chunk - 1) / p.chunk;
    const int BNX = R <= 16 ? 16 : 32;
    CUtensorMap tw, tx;
    int rc;
    if ((rc = br_make_tmap_2d_bf16(&tw, W, N, K, ldw, BM))) return rc;
    if ((rc = br_make_tmap_2d_bf16(&tx, X, R, K, ldx, BNX))) return rc;
    CUtensorMap tp = tw;
    p.pf_on = 0;
    if (prefetch && prefetch->W && prefetch->unit_hi > prefetch->unit_lo) {
        if ((rc = br_make_l2_prefetch(prefetch, &tp, &p.pf.KB, &p.pf.units, &p.pf.chunk, &p.pf.n_chunks, &p.pf.a, &p.pf.b))) return rc;
        p.pf_on = 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (R <= 8) return launch<16, 8>(tw, tx, tp, p, grid, st);
    return BNX == 16 ? launch<16, 16>(tw, tx, tp, p, grid, st) : launch<32, 32>(tw, tx, tp, p, grid, st);
}


/* profiling aid: [n_launches, 160, 8] int64 %globaltimer stamps of the next br_skinny_gemm launches (NULL disables):
 * 0 kernel entry, 1 dependency wait passed, 2 prologue done (barriers initialised), 3 first accumulator, 4 last partial published, 5 reduction loads done,
 * 6 reducer epilogue done, 7 CTA done */
int br_skinny_debug(long long* buf) { g_sk_dbg = buf; g_sk_dbg_slot = 0; return BR_OK; }

static long long* g_chain_dbg = nullptr;
/* profiling aid: [n_sms, 32] int64 %globaltimer stamps of the next chain launches (NULL disables) */
int br_skinny_chain_debug(long long* buf) { g_chain_dbg = buf; return BR_OK; }

int br_skinny_chain(const br_skinny_phase* phases, int n_phases, int R, float eps, void* scratch, void* stream) {
    BR_CHECK_ARG(n_phases >= 1 && n_phases <= CHAIN_MAX && R >= 1 && R <= 32 && scratch, "skinny_chain: 1..%d phases, R in [1, 32]", CHAIN_MAX);
    ChainParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.n_phases = n_phases;
    cp.dbg = g_chain_dbg;
    const int BNX = R <= 16 ? 16 : 32;
    const int grid = br_num_sms();                         // every phase uses the full grid: the barrier counts gridDim.x arrivals
    float* part = (float*)scratch;
    cp.gbar = (int*)(part + (int64_t)br_num_sms() * 2 * 32 * BM);
    for (int i = 0; i < n_phases; ++i) {
        const br_skinny_phase& h = phases[i];
        BR_CHECK_ARG(h.N % 16 == 0 && h.K % 8 == 0 && h.ldx % 8 == 0 && h.ldw % 8 == 0, "skinny_chain[%d]: N %% 16, K %% 8, ld %% 8", i);
        BR_CHECK_ARG(h.mode >= 0 && h.mode <= 3 && !(h.mode == 1 && !h.residual) && !(h.sumsq_out && h.mode >= 2), "skinny_chain[%d]: bad mode", i);
        SkParams& p = cp.ph[i].p;
        p.R = R; p.N = h.N; p.K = h.K; p.mode = h.mode; p.out = h.out; p.ldo = h.ldo; p.res = (const bf16*)h.residual; p.ldr = h.ldr;
        p.scratch = part; p.counters = cp.gbar + 16;
        p.sumsq_in = h.sumsq_in; p.sumsq_in_n = h.sumsq_in_n; p.sumsq_out = h.sumsq_out; p.eps = eps; p.dbg = nullptr; p.dbg_slot = 0; p.w_evict_first = 0;
        p.tiles_n = (h.N + BM - 1) / BM; p.KB = (h.K + BK - 1) / BK; p.units = p.tiles_n * p.KB;
        p.chunk = (p.units + grid - 1) / grid;
        int rc;
        if ((rc = br_make_tmap_2d_bf16(&cp.ph[i].tmW, h.W, h.N, h.K, h.ldw, BM))) return rc;
        if ((rc = br_make_tmap_2d_bf16(&cp.ph[i].tmX, h.X, R, h.K, h.ldx, BNX))) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;      // barrier words gbar[0..1] are zero between launches (self-resetting)
    return BNX == 16 ? launch_chain<16>(cp, grid, st) : launch_chain<32>(cp, grid, st);
}

}  // extern "C"
